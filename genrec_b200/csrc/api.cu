// genrec_b200 - C ABI (include/genrec_b200.h): argument checking, buffer carving and kernel orchestration.
// Nothing here allocates or synchronises; every kernel goes onto the caller's stream.
#include "../../include/genrec_b200.h"

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <initializer_list>
#include <map>
#include <mutex>
#include <type_traits>
#include <utility>

#include "attn_hstu.cuh"
#include "attn_hstu_extend.cuh"
#include "attn_sasrec.cuh"
#include "attn_t5.cuh"
#include "attn_buckets.cuh"
#include "beam.cuh"
#include "common.cuh"
#include "dp_adam.cuh"
#include "exact_f32.cuh"
#include "rowwise.cuh"
#include "rq_argmin.cuh"
#include "rq_sinkhorn.cuh"
#include "tc_gemm.cuh"
#include "tc_ce.cuh"
#include "tc_tn_group.cuh"
#include <cstdlib>

using namespace grb;

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

#define GRB_CUDA(expr)                                                                                  \
    do {                                                                                                \
        cudaError_t _e = (expr);                                                                        \
        if (_e != cudaSuccess) return fail(GRB_ECUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
    } while (0)
#define GRB_REQUIRE(cond, ...)                            \
    do {                                                  \
        if (!(cond)) return fail(GRB_EINVAL, __VA_ARGS__); \
    } while (0)
#define GRB_TRY(expr)          \
    do {                       \
        int _r = (expr);       \
        if (_r != 0) return _r; \
    } while (0)

inline size_t align_up(size_t v, size_t a = 256) { return (v + a - 1) / a * a; }
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int current_device() {
    int dev = 0;
    cudaGetDevice(&dev);
    return dev;
}
int sm_count() {     // per device ordinal: a process may drive several GPUs
    static int n[64] = {0};
    const int dev = current_device() & 63;
    if (n[dev] == 0) {
        int v = 0;
        cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
        n[dev] = v > 0 ? v : 132;
    }
    return n[dev];
}
// 256-thread CTAs for n items, at most per_sm CTAs per SM (the grid-stride kernels loop over the rest)
unsigned capped_blocks(size_t n, int per_sm = 16) {
    const size_t need = (n + 255) / 256, cap = (size_t)sm_count() * per_sm;
    return (unsigned)(need < 1 ? 1 : (need < cap ? need : cap));
}
// bump allocator of the carved layouts: every buffer starts on a 256-byte boundary; with a null base only the size is counted
struct Carver {
    char* base;
    size_t off = 0;
    template <class T>
    T* take(size_t bytes) {
        T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += align_up(bytes);
        return p;
    }
};
// head-dim dispatch of the attention kernels: f(integral_constant DH) for DH = 32 or 64 (check_dims admits nothing else)
template <class F>
int with_head_dim(int dh, F&& f) {
    if (dh == 32) return f(std::integral_constant<int, 32>{});
    return f(std::integral_constant<int, 64>{});
}
// the row kernels are instantiated per D: f(integral_constant D) launches one for D = 64, 128 or 256
template <class F>
int with_row_dim(int D, F&& f) {
    if (D == 64) f(std::integral_constant<int, 64>{});
    else if (D == 128) f(std::integral_constant<int, 128>{});
    else if (D == 256) f(std::integral_constant<int, 256>{});
    else return fail(GRB_EINVAL, "row kernels support D in {64,128,256}, got %d", D);
    GRB_CUDA(cudaGetLastError());
    return 0;
}
int row_grid(int T) {
    int need = (T + ROW_THREADS / 32 - 1) / (ROW_THREADS / 32);
    int cap = sm_count() * 8;
    return need < cap ? (need < 1 ? 1 : need) : cap;
}
int row_bwd_grid(int T) {
    const int need = (T + ROW_THREADS / 32 - 1) / (ROW_THREADS / 32), cap = sm_count() * 3;
    return need < cap ? (need < 1 ? 1 : need) : cap;
}
// grids of the column-sum kernels (their partial scratch is sized from them)
dim3 colsum_grid(int T, int N) {
    const int cx = (N + 255) / 256, maxy = (T + 63) / 64;
    int cy = (4 * sm_count() + cx - 1) / cx;
    cy = cy > maxy ? maxy : cy;
    return dim3(cx, cy < 1 ? 1 : cy);
}
dim3 cast_colsum_grid(int T, int D) {
    const int cx = (D + 127) / 128, maxy = (T + 31) / 32;
    int cy = (8 * sm_count() + cx - 1) / cx;
    cy = cy > maxy ? maxy : cy;
    return dim3(cx, cy < 1 ? 1 : cy);
}
size_t attn_dw_part_floats(int B, int L, int H) { return (size_t)2 * H * B * ((L + ATT_BLK - 1) / ATT_BLK) * 64; }
// the ordered sum of the per-CTA partials a kernel left in `part` (common.cuh det_store, layout [group][member][W]): group g,
// element i -> out[g / gpo][(g % gpo) * gstride + i * estride] when that index < len[g / gpo]
struct DetOut {
    float* out;
    int len;
};
int det_finish(const float* part, int ngroups, int nmembers, int W, int gpo, int gstride, int estride, std::initializer_list<DetOut> outs,
               cudaStream_t st) {
    DetFinishArgs f;
    memset(&f, 0, sizeof(f));
    f.part = part; f.ngroups = ngroups; f.nmembers = nmembers; f.W = W; f.gpo = gpo; f.gstride = gstride; f.estride = estride;
    int k = 0;
    for (const DetOut& o : outs) { f.out[k] = o.out; f.len[k] = o.len; ++k; }
    const unsigned blocks = (unsigned)(((size_t)ngroups * W * 32 + 255) / 256);
    launch_k(det_finish_kernel, blocks, 256, 0, st, f);
    GRB_CUDA(cudaGetLastError());
    return 0;
}

// ---- GEMMs: the wgmma/TMA kernel of tc_gemm.cuh with a fused epilogue.  A is K contiguous; B_MN = 0 -> B K contiguous,
//      1 -> N contiguous.
// z = x W^T + b ; act: 0 none, 1 silu, 2 relu   (NT)
cudaError_t gemm_bias_act(int act, const bf16* x, const bf16* w, const float* bias, bf16* z, bf16* a, int M, int N, int K, const Dropout& drop,
                          cudaStream_t st) {
    if (act == 0) return launch_tc_gemm<0>(x, w, M, N, K, K, K, TcEpiBiasAct<0>{bias, N, drop}, z, nullptr, N, sm_count(), st);
    if (act == 1) return launch_tc_gemm<0>(x, w, M, N, K, K, K, TcEpiBiasAct<1>{bias, N, drop}, z, a, N, sm_count(), st);
    return launch_tc_gemm<0>(x, w, M, N, K, K, K, TcEpiBiasAct<2>{bias, N, drop}, z, a, N, sm_count(), st);
}
// y = res + drop(x W^T + b) (* row_scale)   (NT)
cudaError_t gemm_bias_res(const bf16* x, const bf16* w, const float* bias, const float* res, const float* row_scale, float* y, int M, int N,
                          int K, const Dropout& drop, cudaStream_t st) {
    return launch_tc_gemm<0>(x, w, M, N, K, K, K, TcEpiBiasResidual{bias, res, row_scale, N, drop}, y, nullptr, N, sm_count(), st);
}
// g[M,N] = dropmask(dy[M,K] W[K,N]) * act'(z)   (NN) ; act 1 silu, 2 relu
cudaError_t gemm_dact(int act, const bf16* dy, const bf16* w, const bf16* z, bf16* g, int M, int N, int K, const Dropout& drop, cudaStream_t st) {
    if (act == 1) return launch_tc_gemm<1>(dy, w, M, N, K, K, N, TcEpiDAct<1>{z, N, drop}, g, nullptr, N, sm_count(), st);
    return launch_tc_gemm<1>(dy, w, M, N, K, K, N, TcEpiDAct<2>{z, N, drop}, g, nullptr, N, sm_count(), st);
}
// out[M,N] fp32 = scale * A[M,K] B[K,N] (+ res)   (NN)
cudaError_t gemm_nn_f32(const bf16* A, const bf16* B, float* out, const float* res, float scale, int M, int N, int K, int lda, int ldb,
                        cudaStream_t st) {
    return launch_tc_gemm<1>(A, B, M, N, K, lda, ldb, TcEpiF32{res, N, scale}, out, nullptr, N, sm_count(), st);
}

// ---- carved layouts ------------------------------------------------------------------------------------------
struct LayerSaved {
    bf16 *xb, *zp, *P, *O, *xn, *z1, *hact;
    float *st1, *x1, *st2;
    size_t bytes;
};
LayerSaved carve_saved(void* base, size_t T, size_t D) {
    LayerSaved s;
    Carver c{static_cast<char*>(base)};
    s.xb = c.take<bf16>(T * D * 2);
    s.zp = c.take<bf16>(T * 4 * D * 2);
    s.P = c.take<bf16>(T * 4 * D * 2);
    s.O = c.take<bf16>(T * D * 2);
    s.st1 = c.take<float>(T * 2 * 4);
    s.x1 = c.take<float>(T * D * 4);
    s.xn = c.take<bf16>(T * D * 2);
    s.st2 = c.take<float>(T * 2 * 4);
    s.z1 = c.take<bf16>(T * 4 * D * 2);
    s.hact = c.take<bf16>(T * 4 * D * 2);
    s.bytes = c.off;
    return s;
}
struct LayerWork {
    bf16 *dyb, *dz1, *dO, *dzp;
    float *dxn, *dx1;
    // scratch of the ordered cross-CTA sums: weight-gradient split-K tiles, bias column sums, LayerNorm and bias-table gradients
    float *part_tn, *part_colsum, *part_cast, *part_ln, *part_attn;
    size_t bytes;
};
void layer_tn_specs(TnSpec (&specs)[3], const bf16* dyb, const bf16* hact, const bf16* dz1, const bf16* xn, const bf16* dzp, const bf16* xb,
                    float* dw2, float* dw1, float* dwp, int T, int D) {
    specs[0] = {dyb, hact, dw2, D, 4 * D, T, D, 4 * D, 4 * D};   // dW2 += dyb^T h
    specs[1] = {dz1, xn, dw1, 4 * D, D, T, 4 * D, D, D};         // dW1 += dz1^T xn
    specs[2] = {dzp, xb, dwp, 4 * D, D, T, 4 * D, D, D};         // dWp += dzp^T xb
}
LayerWork carve_work(void* base, const grb_hstu_dims* d) {
    const size_t T = (size_t)d->B * d->L, D = d->D;
    LayerWork w;
    Carver c{static_cast<char*>(base)};
    w.dyb = c.take<bf16>(T * D * 2);
    w.dz1 = c.take<bf16>(T * 4 * D * 2);
    w.dxn = c.take<float>(T * D * 4);
    w.dx1 = c.take<float>(T * D * 4);
    w.dO = c.take<bf16>(T * D * 2);
    w.dzp = c.take<bf16>(T * 4 * D * 2);
    TnSpec specs[3];
    layer_tn_specs(specs, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, (int)T, (int)D);
    w.part_tn = c.take<float>(tn_part_floats(specs, 3, sm_count()) * 4);
    const dim3 cg = colsum_grid((int)T, 4 * (int)D), kg = cast_colsum_grid((int)T, (int)D);
    w.part_colsum = c.take<float>((size_t)cg.x * cg.y * 256 * 4);
    w.part_cast = c.take<float>((size_t)kg.x * kg.y * 128 * 4);
    w.part_ln = c.take<float>((size_t)4 * row_grid((int)T) * D * 4);
    w.part_attn = c.take<float>(attn_dw_part_floats(d->B, d->L, d->H) * 4);
    w.bytes = c.off;
    return w;
}

int check_dims(const grb_hstu_dims* d) {
    GRB_REQUIRE(d != nullptr, "dims is null");
    GRB_REQUIRE(d->B > 0 && d->L > 0 && d->H > 0, "B, L, H must be positive (B=%d L=%d H=%d)", d->B, d->L, d->H);
    GRB_REQUIRE(d->D == 64 || d->D == 128 || d->D == 256, "embed_dim %d unsupported (64, 128, 256)", d->D);
    GRB_REQUIRE(d->D % d->H == 0, "embed_dim %% num_heads != 0");
    int dh = d->D / d->H;
    GRB_REQUIRE(dh == 32 || dh == 64, "head_dim %d unsupported (32, 64)", dh);
    GRB_REQUIRE(d->npos >= 1 && d->npos <= ATT_MAX_BUCKETS, "num_position_buckets %d out of range [1,64]", d->npos);
    GRB_REQUIRE(d->ntime >= 0 && d->ntime <= ATT_MAX_BUCKETS, "num_time_buckets %d out of range [0,64]", d->ntime);
    GRB_REQUIRE(d->L <= 16384, "seq_len %d too long", d->L);
    GRB_REQUIRE(d->dropout_p >= 0.f && d->dropout_p < 1.f, "dropout_p out of range");
    return 0;
}
int check_layer_params(const grb_hstu_layer_params* p) {
    GRB_REQUIRE(p != nullptr, "null argument");
    GRB_REQUIRE(p->proj_w && p->proj_b && p->pos_table && p->ln1_g && p->ln1_b && p->ffn1_w && p->ffn1_b && p->ffn2_w &&
                    p->ffn2_b && p->ln2_g && p->ln2_b, "null parameter pointer");
    GRB_REQUIRE(aligned16(p->proj_w) && aligned16(p->ffn1_w) && aligned16(p->ffn2_w), "weights must be 16-byte aligned");
    return 0;
}
int check_seq(const grb_hstu_dims* d, const grb_hstu_seq* s) {
    GRB_REQUIRE(s != nullptr && s->bias_index, "null sequence metadata: the attention kernels need bias_index");
    GRB_REQUIRE(s->ld_index >= d->L && s->ld_index % 8 == 0 && aligned16(s->bias_index),
                "bias_index must be 16-byte aligned with a pitch that is a multiple of 8 and >= L");
    return 0;
}

// opt in to > 48 KB dynamic shared memory once per (kernel, high-water mark): no runtime call on the steady-state path,
// in particular none while a CUDA graph is being captured after warm-up.
template <class Kern>
int set_smem(Kern k, size_t bytes) {
    static std::mutex mu;
    static std::map<std::pair<int, const void*>, size_t> high_water;  // keyed by (device, kernel address): the attribute is per device
    std::lock_guard<std::mutex> lock(mu);
    size_t& hw = high_water[std::make_pair(current_device(), reinterpret_cast<const void*>(k))];
    if (hw < 48 * 1024) hw = 48 * 1024;
    if (bytes > hw) {
        GRB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
        hw = bytes;
    }
    return 0;
}

// the bias tables without the index matrix (bias_index null, ldix 0)
HstuBiasArgs make_attn_bias(const grb_hstu_dims* d, const float* pos_table, const float* time_table, int has_time, int pos_uniform,
                            int pos_bucket0) {
    HstuBiasArgs b;
    memset(&b, 0, sizeof(b));
    // uniform position buckets (the reference's behaviour) collapse to ONE effective bucket: the index matrix was built with
    // npos = 1, the tables shrink to 65 entries and the pointers are offset to the single live row of the [npos, H] table
    b.wpos = pos_table + (pos_uniform ? (size_t)pos_bucket0 * d->H : 0);
    const bool timed = time_table != nullptr && has_time && d->ntime > 0;
    b.wtime = timed ? time_table : nullptr;
    b.pos_uniform = pos_uniform;
    b.npos = pos_uniform ? 1 : d->npos;
    b.ntime = timed ? d->ntime : 0;
    b.time_bins = att_time_bins(timed, pos_uniform != 0, b.ntime);
    return b;
}
HstuBiasArgs make_attn_bias(const grb_hstu_dims* d, const float* pos_table, const float* time_table, const grb_hstu_seq* s) {
    HstuBiasArgs b = make_attn_bias(d, pos_table, time_table, s->has_time, s->pos_uniform, s->pos_bucket0);
    b.bias_index = s->bias_index;
    b.ldix = s->ld_index;
    return b;
}
// P: [T, 4D] bf16 U | V | Q | K ; O: [T, D] bf16 output, written by the forward only
HstuAttnArgs make_attn_args(const grb_hstu_dims* d, const float* pos_table, const float* time_table, const grb_hstu_seq* s, const bf16* P,
                            bf16* O) {
    HstuAttnArgs a;
    memset(&a, 0, sizeof(a));
    const int D = d->D;
    a.q = P + 2 * D; a.k = P + 3 * D; a.v = P + D;
    a.ldq = a.ldk = a.ldv = 4 * D;
    a.B = d->B; a.L = d->L; a.H = d->H;
    a.bias = make_attn_bias(d, pos_table, time_table, s);
    a.o = O; a.ldo = D;
    return a;
}
// the backward's side of the attention arguments.  zp (nullable) and dzp are [T, 4D] bf16 in U | V | Q | K order: the
// pre-activations and their gradients.  With uniform position buckets dpos is pointed at the single live row of the table.
int set_attn_bwd_args(HstuAttnArgs& a, const grb_hstu_dims* d, const grb_hstu_seq* s, const bf16* dO, const bf16* zp, bf16* dzp,
                      float* dpos, float* dtime, float* part) {
    GRB_REQUIRE(a.bias.wtime == nullptr || dtime != nullptr, "time_table gradient pointer is null");
    const int D = d->D;
    a.d_o = dO; a.lddo = D;
    a.zq = zp ? zp + 2 * D : nullptr; a.zk = zp ? zp + 3 * D : nullptr; a.zv = zp ? zp + D : nullptr; a.ldz = 4 * D;
    a.dq = dzp + 2 * D; a.dk = dzp + 3 * D; a.dv = dzp + D; a.lddq = 4 * D;
    a.dwpos = dpos + (s->pos_uniform ? (size_t)s->pos_bucket0 * d->H : 0);
    a.dwtime = dtime;
    a.dw_part = part;
    return 0;
}

template <int DH>
int launch_hstu_attn_fwd(const HstuAttnArgs& a, cudaStream_t st) {
    size_t smem = sizeof(AttSmem<DH, 1>) + align_up((size_t)(a.bias.npos * 64 + 1) * 4, 16);
    GRB_TRY(set_smem(hstu_attn_fwd_kernel<DH>, smem));
    dim3 grid((a.L + ATT_BLK - 1) / ATT_BLK, a.H, a.B);
    launch_k(hstu_attn_fwd_kernel<DH>, grid, ATT_THREADS, smem, st, a);
    GRB_CUDA(cudaGetLastError());
    return 0;
}
// Fork/join helper: a non-blocking stream and its two events, created on first use, i.e. during warm-up, never while a CUDA graph
// is being captured.  Event fork / join also pulls the side stream into a capture.
struct SideStream {
    cudaStream_t s = nullptr;
    cudaEvent_t fork = nullptr, join = nullptr;
    bool ok = false, pending = false;
    // run `launch(s)` after everything enqueued on `st` so far; returns 0 / error code
    template <class F>
    int run(cudaStream_t st, F&& launch) {
        if (!ok) {
            GRB_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
            GRB_CUDA(cudaEventCreateWithFlags(&fork, cudaEventDisableTiming));
            GRB_CUDA(cudaEventCreateWithFlags(&join, cudaEventDisableTiming));
            ok = true;
        }
        GRB_CUDA(cudaEventRecord(fork, st));
        GRB_CUDA(cudaStreamWaitEvent(s, fork, 0));
        GRB_TRY(launch(s));
        GRB_CUDA(cudaEventRecord(join, s));
        pending = true;
        return 0;
    }
    // make `st` wait for everything run() has enqueued since the last join
    int join_into(cudaStream_t st) {
        if (pending) {
            GRB_CUDA(cudaStreamWaitEvent(st, join, 0));
            pending = false;
        }
        return 0;
    }
};
// dQ and dK/dV are independent, both latency-bound at low occupancy: dQ runs on this stream beside dK/dV.  Not the deferred
// stream, where dQ would queue behind the weight-gradient GEMMs.  The backward runs on the autograd thread: one instance per
// calling thread and device.
SideStream& attn_side_stream() {
    static thread_local SideStream ss[64];
    return ss[current_device() & 63];
}
// ---- deferred weight gradients.  dW / dE GEMMs are not on the critical path of a training step: nothing reads them before the
// optimizer.  With grb_set_defer_weight_grads(1) they go to a per-device side stream, forked where their operands are ready and
// joined by grb_join_deferred() (FlatAdam.step calls it), so they fill the SM tails of the epilogue-bound GEMMs and run next to the
// issue-bound attention kernels; the 620 MB dlogits stream of the head's dE GEMM overlaps the last block's backward.  The CALLER keeps
// the operand buffers (layer workspace, saved blob, head workspace) alive until the join.
std::mutex g_defer_mu;
bool g_defer_on = false;
SideStream& defer_stream() {
    static SideStream ds[64];
    return ds[current_device() & 63];
}
template <class F>
int defer_run(cudaStream_t st, F&& launch) {
    std::lock_guard<std::mutex> lock(g_defer_mu);
    return defer_stream().run(st, launch);
}
int join_pending(cudaStream_t st) {
    std::lock_guard<std::mutex> lock(g_defer_mu);
    return defer_stream().join_into(st);
}
// launch(side stream) with the deferred schedule on, launch(st) without it
template <class F>
int run_maybe_deferred(cudaStream_t st, F&& launch) {
    if (g_defer_on) return defer_run(st, launch);
    return launch(st);
}

template <int DH>
int launch_hstu_attn_bwd(const HstuAttnArgs& a, cudaStream_t st) {
    dim3 grid((a.L + ATT_BLK - 1) / ATT_BLK, a.H, a.B);
    size_t posb = align_up((size_t)(a.bias.npos * 64 + 1) * 4, 16);  // combined bias table
    size_t smem_q = sizeof(AttSmem<DH>) + posb;
    GRB_TRY(set_smem(hstu_attn_bwd_dq_kernel<DH>, smem_q));
    SideStream& ss = attn_side_stream();
    GRB_TRY(ss.run(st, [&](cudaStream_t side) -> int {
        launch_k(hstu_attn_bwd_dq_kernel<DH>, grid, ATT_THREADS, smem_q, side, a);
        GRB_CUDA(cudaGetLastError());
        return 0;
    }));
    const bool has_time = a.bias.wtime != nullptr && a.bias.ntime > 0, pos_uni = a.bias.pos_uniform != 0;
    size_t smem_k = sizeof(AttSmemKV<DH>) + posb +
                    (size_t)4 * (att_time_bins(has_time, pos_uni, a.bias.ntime) + (pos_uni ? 0 : a.bias.npos + 1)) * 32 * sizeof(float);
    const int nmem = (int)(grid.x * grid.z), ngroups = has_time && a.dwtime ? 2 * a.H : a.H;
    GRB_REQUIRE((pos_uni || a.bias.npos <= 64) && a.bias.ntime <= 64, "attention backward: at most 64 position / time buckets");
    auto go = [&](auto kern) -> int {
        GRB_TRY(set_smem(kern, smem_k));
        launch_k(kern, grid, ATT_THREADS, smem_k, st, a, (int)posb);
        return 0;
    };
    if (has_time && pos_uni) GRB_TRY(go(hstu_attn_bwd_dkdv_kernel<DH, true, true>));
    else if (has_time) GRB_TRY(go(hstu_attn_bwd_dkdv_kernel<DH, true, false>));
    else if (pos_uni) GRB_TRY(go(hstu_attn_bwd_dkdv_kernel<DH, false, true>));
    else GRB_TRY(go(hstu_attn_bwd_dkdv_kernel<DH, false, false>));
    // groups h < H: position buckets of head h ; H + h: time buckets of head h ; element = bucket.  With uniform positions
    // the caller has already pointed dwpos at the single live row.
    float* pos_out = a.dwpos;
    const int pos_len = pos_uni ? a.H : a.bias.npos * a.H;
    if (ngroups > a.H) GRB_TRY(det_finish(a.dw_part, ngroups, nmem, 64, a.H, 1, a.H, {{pos_out, pos_len}, {a.dwtime, a.bias.ntime * a.H}}, st));
    else GRB_TRY(det_finish(a.dw_part, ngroups, nmem, 64, a.H, 1, a.H, {{pos_out, pos_len}}, st));
    GRB_CUDA(cudaGetLastError());
    GRB_TRY(ss.join_into(st));
    return 0;
}

int cast_bf16(const float* in, bf16* out, size_t n, int D, const Dropout& drop, const float* row_scale, cudaStream_t st) {
    GRB_REQUIRE(D > 0 && D % 4 == 0 && n % (size_t)D == 0, "cast needs rows of a multiple-of-4 length D");
    launch_k(cast_f32_bf16_kernel, capped_blocks(n / 4), 256, 0, st, in, out, n, D, drop, row_scale);
    GRB_CUDA(cudaGetLastError());
    return 0;
}
// part: cast_colsum_grid(T, D).x * .y * 128 floats of scratch for the ordered sum
int cast_colsum(const float* in, bf16* out, int T, int D, const Dropout& drop, float* colsum_out, float* part, cudaStream_t st) {
    GRB_REQUIRE(D > 0 && D % 4 == 0, "cast needs rows of a multiple-of-4 length D");
    const dim3 grid = cast_colsum_grid(T, D);
    launch_k(cast_colsum_f32_bf16_kernel, grid, 256, 0, st, in, out, T, D, drop, part);
    GRB_CUDA(cudaGetLastError());
    GRB_TRY(det_finish(part, grid.x, grid.y, 128, grid.x, 128, 1, {{colsum_out, D}}, st));
    return 0;
}
// part: colsum_grid(T, N).x * .y * 256 floats of scratch for the ordered sum
int colsum(const bf16* in, int T, int N, int ld, float* out, float* part, cudaStream_t st) {
    if (N % 8 != 0 || ld % 8 != 0) return fail(GRB_EINVAL, "colsum needs N and ld to be multiples of 8");
    const dim3 grid = colsum_grid(T, N);
    launch_k(colsum_bf16_kernel, grid, 256, 0, st, in, T, N, ld, part);
    GRB_CUDA(cudaGetLastError());
    GRB_TRY(det_finish(part, grid.x, grid.y, 256, grid.x, 256, 1, {{out, N}}, st));
    return 0;
}
// dx = (res ? res : 0) + LNbwd(dy) ; dg += , db += in a fixed order.  a.part: 2 * row_bwd_grid(T) * D floats of scratch
int ln_backward(const LnBwdArgs& a, cudaStream_t st) {
    GRB_TRY(with_row_dim(a.D, [&](auto DC) { launch_k(ln_bwd_kernel<DC / 64>, row_bwd_grid(a.T), ROW_THREADS, 0, st, a); }));
    return det_finish(a.part, 2, row_bwd_grid(a.T), a.D, 1, 0, 1, {{a.dg, a.D}, {a.db, a.D}}, st);
}

// ---- cached incremental inference (attn_hstu_extend.cuh)
// keys per CTA of the chunk attention: enough key splits that B * H * query tiles * splits reaches about four CTAs per SM (one
// new item per user must still fill the GPU), at least one 64-key tile each.  A function of the shapes and the capacity only, so
// the grid is the same on every call and a captured graph stays valid while the lengths grow on the device.
int extend_split(const grb_hstu_dims* d, int capacity) {
    const long long base = (long long)d->B * d->H * ((d->L + ATT_BLK - 1) / ATT_BLK);
    const long long want = (4LL * sm_count() + base - 1) / base;
    const int per = (int)((capacity + want - 1) / want);
    return (per + ATT_BLK - 1) / ATT_BLK * ATT_BLK;
}
int check_extend(const grb_hstu_dims* d, int capacity) {
    GRB_TRY(check_dims(d));
    GRB_REQUIRE(capacity >= 1 && capacity <= 16384, "cache capacity %d out of range [1, 16384]", capacity);
    GRB_REQUIRE(d->dropout_p == 0.f, "the cached extend is inference only: dropout_p must be 0");
    GRB_REQUIRE((long long)d->B * ((d->L + ATT_BLK - 1) / ATT_BLK) <= 65535, "B * ceil(n / 64) = %lld exceeds 65535",
                (long long)d->B * ((d->L + ATT_BLK - 1) / ATT_BLK));
    return 0;
}
// workspace: the forward's activation layout for the chunk's B * n rows, then the [splits, B * n, D] fp32 attention partials
struct ExtendWork {
    LayerSaved sv;
    float* part;
    size_t bytes;
};
ExtendWork carve_extend(void* base, const grb_hstu_dims* d, int capacity) {
    const size_t T = (size_t)d->B * d->L;
    ExtendWork w;
    w.sv = carve_saved(base, T, d->D);
    const int split = extend_split(d, capacity);
    const size_t nsplit = (capacity + split - 1) / split;
    w.part = base ? reinterpret_cast<float*>(static_cast<char*>(base) + w.sv.bytes) : nullptr;
    w.bytes = w.sv.bytes + align_up(nsplit * T * d->D * 4);
    return w;
}
template <int DH, bool UNIFORM, bool TIMED>
int launch_attn_extend(const HstuExtendArgs& a, int nsplit, cudaStream_t st) {
    const size_t smem = sizeof(ExtSmem<DH>) + align_up((size_t)(a.bias.npos * 64 + 1) * 4, 16);
    GRB_TRY(set_smem(hstu_attn_extend_kernel<DH, UNIFORM, TIMED>, smem));
    const dim3 grid(nsplit, a.H, a.B * ((a.n + ATT_BLK - 1) / ATT_BLK));
    launch_k(hstu_attn_extend_kernel<DH, UNIFORM, TIMED>, grid, ATT_THREADS, smem, st, a);
    GRB_CUDA(cudaGetLastError());
    return 0;
}
template <int DH>
int dispatch_attn_extend(const HstuExtendArgs& a, int nsplit, cudaStream_t st) {
    const bool uni = a.pos_bucket == nullptr, timed = a.bias.wtime != nullptr;
    if (uni && timed) return launch_attn_extend<DH, true, true>(a, nsplit, st);
    if (uni) return launch_attn_extend<DH, true, false>(a, nsplit, st);
    if (timed) return launch_attn_extend<DH, false, true>(a, nsplit, st);
    return launch_attn_extend<DH, false, false>(a, nsplit, st);
}

// Where one layer's cached K | V lives: the dense cache (users and page table null, page_size = capacity) or a pool.
struct ExtendKv {
    bf16* kv;                  // this layer's rows [pages * page_size, 2D]
    const long long* ts;       // [pages * page_size]
    const long long* users;    // [B] or null
    KvPages pg;
    int cap;                   // most items a user can hold
};
int check_pool(const grb_hstu_pool* p) {
    GRB_REQUIRE(p != nullptr, "null pool");
    GRB_REQUIRE(p->page_size >= ATT_BLK && p->page_size % ATT_BLK == 0, "page_size %d must be a positive multiple of %d", p->page_size, ATT_BLK);
    GRB_REQUIRE(p->max_items >= 1 && p->max_items <= 16384, "pool max_items %d out of range [1, 16384]", p->max_items);
    GRB_REQUIRE(p->max_users > 0 && p->num_pages > 0 && p->num_layers > 0, "bad pool shape max_users=%d num_pages=%d num_layers=%d",
                p->max_users, p->num_pages, p->num_layers);
    return 0;
}
inline int pool_pt_ld(const grb_hstu_pool* p) { return (p->max_items + p->page_size - 1) / p->page_size; }
HstuPoolArgs pool_args(const grb_hstu_pool* p, const int64_t* users, int B) {
    HstuPoolArgs a;
    memset(&a, 0, sizeof(a));
    a.users = reinterpret_cast<const long long*>(users); a.B = B;
    a.max_users = p->max_users; a.max_items = p->max_items; a.num_pages = p->num_pages;
    a.page_table = p->page_table; a.pt_ld = pool_pt_ld(p); a.page_size = p->page_size;
    a.len = p->lengths; a.overflow = p->overflow; a.free_stack = p->free_stack; a.free_top = p->free_top;
    a.errors = p->errors; a.row_of = p->row_of;
    return a;
}

// steps 1-2 of the block: xb = bf16(x) (GEMM operand; also the dWp operand in backward) ; P = silu(x Wp^T + bp) -> [U | V | Q | K]
//                                                                                            (hstu.py:234-235)
int block_steps_in(const grb_hstu_layer_params* p, const float* x, const LayerSaved& sv, int T, int D, cudaStream_t st) {
    const Dropout nodrop = make_dropout(0.f, 0, 0);
    GRB_TRY(cast_bf16(x, sv.xb, (size_t)T * D, D, nodrop, nullptr, st));
    GRB_CUDA(gemm_bias_act(1, sv.xb, (const bf16*)p->proj_w, p->proj_b, sv.zp, sv.P, T, 4 * D, D, nodrop, st));
    return 0;
}
// steps 4-6 of the block, after the attention has written O
int block_steps_out(const grb_hstu_layer_params* p, const float* x, float* y, const LayerSaved& sv, int T, int D, const Dropout& drop_gate,
                    const Dropout& drop_hid, const Dropout& drop_out, cudaStream_t st) {
    // 4. x1 = x + drop(LN1(O) * U) ; xn = LN2(x1)                                            (hstu.py:271-278)
    LnGateFwdArgs a{sv.O, D, sv.P, 4 * D, x, p->ln1_g, p->ln1_b, p->ln2_g, p->ln2_b, sv.x1, sv.xn, sv.st1, sv.st2, T, D, 1e-5f, drop_gate};
    GRB_TRY(with_row_dim(D, [&](auto DC) { launch_k(ln_gate_fwd_kernel<DC / 64>, row_grid(T), ROW_THREADS, 0, st, a); }));
    // 5. h = drop(silu(xn W1^T + b1))                                                        (hstu.py:210-212)
    GRB_CUDA(gemm_bias_act(1, sv.xn, (const bf16*)p->ffn1_w, p->ffn1_b, sv.z1, sv.hact, T, 4 * D, D, drop_hid, st));
    // 6. y = x1 + drop(h W2^T + b2)                                                          (hstu.py:213-214, :278)
    GRB_CUDA(gemm_bias_res(sv.hact, (const bf16*)p->ffn2_w, p->ffn2_b, sv.x1, nullptr, y, T, D, 4 * D, drop_out, st));
    return 0;
}

// the steps of grb_hstu_layer_forward on the chunk's rows, with the attention against the cache in place of step 3
int layer_extend(const grb_hstu_dims* d, const grb_hstu_layer_params* p, const ExtendKv& c, const int32_t* positions,
                 const uint8_t* pos_bucket, int pos_bucket0, const int64_t* time_thr, const float* x, float* y, void* workspace,
                 cudaStream_t st) {
    GRB_TRY(check_layer_params(p));
    GRB_REQUIRE(pos_bucket != nullptr || (pos_bucket0 >= 0 && pos_bucket0 < d->npos), "pos_bucket0 %d out of range", pos_bucket0);
    const bool timed = d->ntime > 0 && p->time_table != nullptr;
    GRB_REQUIRE(!timed || time_thr != nullptr, "time_thr is null");
    GRB_REQUIRE(aligned16(x) && aligned16(y) && aligned16(workspace) && aligned16(c.kv), "buffers must be 16-byte aligned");
    const int T = d->B * d->L, D = d->D, cap = c.cap;
    ExtendWork w = carve_extend(workspace, d, cap);
    LayerSaved& sv = w.sv;

    GRB_TRY(block_steps_in(p, x, sv, T, D, st));
    {
        const size_t pieces = (size_t)T * (2 * D / 8);
        launch_k(hstu_kv_scatter_kernel, (unsigned)((pieces + 255) / 256), 256, 0, st, (const bf16*)sv.P, (const int*)positions, c.users, T,
                 d->L, D, c.pg, c.kv);
        GRB_CUDA(cudaGetLastError());
    }
    {
        HstuExtendArgs a;
        memset(&a, 0, sizeof(a));
        a.q = sv.P + 2 * D; a.ldq = 4 * D;
        a.kv = c.kv;
        a.ts = c.ts;
        a.users = c.users;
        a.pg = c.pg;
        a.pos = positions;
        a.pos_bucket = pos_bucket;
        a.thr = reinterpret_cast<const long long*>(time_thr);
        a.bias = make_attn_bias(d, p->pos_table, p->time_table, timed, pos_bucket == nullptr, pos_bucket0);
        a.B = d->B; a.n = d->L; a.H = d->H; a.D = D; a.cap = cap;
        a.split = extend_split(d, cap);
        a.part = w.part;
        const int nsplit = (cap + a.split - 1) / a.split;
        GRB_TRY(with_head_dim(D / d->H, [&](auto DH) { return dispatch_attn_extend<DH>(a, nsplit, st); }));
        const size_t quads = (size_t)T * D / 4;
        launch_k(hstu_extend_combine_kernel, (unsigned)((quads + 255) / 256), 256, 0, st, (const float*)w.part, (const int*)positions, T, D,
                 a.split, sv.O);
        GRB_CUDA(cudaGetLastError());
    }
    const Dropout nodrop = make_dropout(0.f, 0, 0);
    return block_steps_out(p, x, y, sv, T, D, nodrop, nodrop, nodrop, st);
}

constexpr uint32_t SITE_GATE = 0, SITE_FFN_HID = 1, SITE_FFN_OUT = 2, SITE_EMBED = 250, SITE_ATTN = 3;
inline uint32_t site_of(int layer, uint32_t which) { return (uint32_t)layer * 8u + which; }

}  // namespace

extern "C" {

const char* grb_last_error(void) { return g_err; }
int grb_version(void) { return 100; }
uint64_t grb_launch_count(void) { return (uint64_t)launch_counter(); }

int grb_check_device(int ordinal) {
    cudaDeviceProp prop;
    cudaError_t e = cudaGetDeviceProperties(&prop, ordinal);
    if (e != cudaSuccess) return fail(GRB_ENODEV, "cudaGetDeviceProperties(%d): %s", ordinal, cudaGetErrorString(e));
    if (prop.major != 9 || prop.minor != 0) return fail(GRB_ENODEV, "device %d is sm_%d%d; this library is built for sm_90a only", ordinal, prop.major, prop.minor);
    return 0;
}

size_t grb_hstu_layer_saved_bytes(const grb_hstu_dims* d) {
    if (check_dims(d)) return 0;
    return carve_saved(nullptr, (size_t)d->B * d->L, d->D).bytes;
}
size_t grb_hstu_layer_workspace_bytes(const grb_hstu_dims* d) {
    if (check_dims(d)) return 0;
    return carve_work(nullptr, d).bytes;
}

int grb_hstu_layer_forward(const grb_hstu_dims* d, const grb_hstu_layer_params* p, const grb_hstu_seq* s, const float* x,
                           float* y, void* saved, void* stream) {
    GRB_TRY(check_dims(d));
    GRB_REQUIRE(x && y && saved, "null argument");
    GRB_TRY(check_layer_params(p));
    GRB_TRY(check_seq(d, s));
    GRB_REQUIRE(aligned16(x) && aligned16(y) && aligned16(saved), "buffers must be 16-byte aligned");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int T = d->B * d->L, D = d->D;
    LayerSaved sv = carve_saved(saved, T, D);

    GRB_TRY(block_steps_in(p, x, sv, T, D, st));
    // 3. O = silu(Q K^T + bias) V, causal + key padding                                      (hstu.py:244-267)
    GRB_TRY(join_pending(st));   // a bias-index matrix built on the side stream (deferred schedule) must be complete
    HstuAttnArgs a = make_attn_args(d, p->pos_table, p->time_table, s, sv.P, sv.O);
    GRB_TRY(with_head_dim(D / d->H, [&](auto DH) { return launch_hstu_attn_fwd<DH>(a, st); }));
    return block_steps_out(p, x, y, sv, T, D, make_dropout(d->dropout_p, d->seed, site_of(d->layer_index, SITE_GATE), d->seed_dev),
                           make_dropout(d->dropout_p, d->seed, site_of(d->layer_index, SITE_FFN_HID), d->seed_dev),
                           make_dropout(d->dropout_p, d->seed, site_of(d->layer_index, SITE_FFN_OUT), d->seed_dev), st);
}

int grb_hstu_layer_backward(const grb_hstu_dims* d, const grb_hstu_layer_params* p, const grb_hstu_seq* s, const float* dy,
                            const void* saved, float* dx, const grb_hstu_layer_grads* g, void* workspace, void* stream) {
    GRB_TRY(check_dims(d));
    GRB_REQUIRE(p && dy && saved && dx && g && workspace, "null argument");
    GRB_TRY(check_seq(d, s));
    GRB_REQUIRE(g->proj_w && g->proj_b && g->pos_table && g->ln1_g && g->ln1_b && g->ffn1_w && g->ffn1_b && g->ffn2_w && g->ffn2_b &&
                    g->ln2_g && g->ln2_b, "null gradient pointer");
    GRB_REQUIRE(aligned16(dy) && aligned16(dx) && aligned16(saved) && aligned16(workspace), "buffers must be 16-byte aligned");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int T = d->B * d->L, D = d->D;
    LayerSaved sv = carve_saved(const_cast<void*>(saved), T, D);
    LayerWork w = carve_work(workspace, d);
    const Dropout drop_out = make_dropout(d->dropout_p, d->seed, site_of(d->layer_index, SITE_FFN_OUT), d->seed_dev);
    const Dropout drop_hid = make_dropout(d->dropout_p, d->seed, site_of(d->layer_index, SITE_FFN_HID), d->seed_dev);
    const Dropout drop_gate = make_dropout(d->dropout_p, d->seed, site_of(d->layer_index, SITE_GATE), d->seed_dev);

    // FFN second linear
    GRB_TRY(cast_colsum(dy, w.dyb, T, D, drop_out, g->ffn2_b, w.part_cast, st));   // dyb = bf16(dropmask(dy)) ; db2 += column sums
    GRB_CUDA(gemm_dact(1, w.dyb, (const bf16*)p->ffn2_w, sv.z1, w.dz1, T, 4 * D, D, drop_hid, st));  // dz1 = dropmask(dyb W2) * silu'(z1)
    // FFN first linear
    // bias gradients are off the critical path too: with deferred weight gradients the column sums run beside the main chain
    auto colsum_4d = [&](const bf16* in, float* out) {
        return run_maybe_deferred(st, [&](cudaStream_t s_) -> int { return colsum(in, T, 4 * D, 4 * D, out, w.part_colsum, s_); });
    };
    GRB_TRY(colsum_4d(w.dz1, g->ffn1_b));
    GRB_CUDA(gemm_nn_f32(w.dz1, (const bf16*)p->ffn1_w, w.dxn, nullptr, 1.f, T, D, 4 * D, 4 * D, D, st));  // dxn = dz1 W1
    // LN2 + residual + gate + LN1
    {
        LnGateBwdArgs a{dy, w.dxn, sv.x1, sv.st1, sv.st2, sv.O, D, sv.P, 4 * D, sv.zp, 4 * D, p->ln1_g, p->ln1_b, p->ln2_g,
                        w.dx1, w.dO, D, w.dzp, 4 * D, g->ln1_g, g->ln1_b, g->ln2_g, g->ln2_b, T, D, drop_gate, w.part_ln};
        GRB_TRY(with_row_dim(D, [&](auto DC) { launch_k(ln_gate_bwd_kernel<DC / 64>, row_grid(T), ROW_THREADS, 0, st, a); }));
        GRB_TRY(det_finish(w.part_ln, 4, row_grid(T), D, 1, 0, 1, {{a.dg1, D}, {a.db1, D}, {a.dg2, D}, {a.db2, D}}, st));
    }
    // attention backward -> gradients w.r.t. the V, Q, K pre-activations
    {
        HstuAttnArgs a = make_attn_args(d, p->pos_table, p->time_table, s, sv.P, sv.O);
        GRB_TRY(set_attn_bwd_args(a, d, s, w.dO, sv.zp, w.dzp, g->pos_table, g->time_table, w.part_attn));
        GRB_TRY(with_head_dim(D / d->H, [&](auto DH) { return launch_hstu_attn_bwd<DH>(a, st); }));
    }
    // projection
    GRB_TRY(colsum_4d(w.dzp, g->proj_b));
    GRB_CUDA(gemm_nn_f32(w.dzp, (const bf16*)p->proj_w, dx, w.dx1, 1.f, T, D, 4 * D, 4 * D, D, st));  // dx = dx1 + dzp Wp
    // the three weight gradients of the layer in ONE grouped launch: dW2 += dyb^T h, dW1 += dz1^T xn, dWp += dzp^T xb
    TnSpec specs[3];
    layer_tn_specs(specs, w.dyb, sv.hact, w.dz1, sv.xn, w.dzp, sv.xb, g->ffn2_w, g->ffn1_w, g->proj_w, T, D);
    return run_maybe_deferred(st, [&](cudaStream_t s_) -> int {
        GRB_CUDA(launch_tc_tn_group(specs, 3, sm_count(), w.part_tn, s_));
        return 0;
    });
}

int grb_hstu_cache_append(const grb_hstu_cache* c, const int64_t* input_ids, const int64_t* timestamps, int n, int32_t* positions,
                          int32_t* last_row, void* stream) {
    GRB_REQUIRE(c && input_ids && positions && last_row, "null argument");
    GRB_REQUIRE(c->timestamps && c->lengths && c->overflow, "null cache pointer");
    GRB_REQUIRE(c->B > 0 && n > 0, "bad shape B=%d n=%d", c->B, n);
    GRB_REQUIRE(c->capacity >= 1 && c->capacity <= 16384, "cache capacity %d out of range [1, 16384]", c->capacity);
    launch_k(hstu_cache_append_kernel, (unsigned)((c->B + 3) / 4), 128, 0, static_cast<cudaStream_t>(stream),
             reinterpret_cast<const long long*>(input_ids), reinterpret_cast<const long long*>(timestamps), (const long long*)nullptr,
             (const int*)nullptr, c->B, n, c->capacity, KvPages{nullptr, 1, c->capacity}, reinterpret_cast<long long*>(c->timestamps),
             c->lengths, c->overflow, positions, last_row);
    GRB_CUDA(cudaGetLastError());
    return 0;
}

int grb_hstu_pool_append(const grb_hstu_pool* pool, const int64_t* users, int B, const int64_t* input_ids, const int64_t* timestamps,
                         int n, int32_t* positions, int32_t* last_row, int32_t* room, void* stream) {
    GRB_TRY(check_pool(pool));
    GRB_REQUIRE(users && input_ids && positions && last_row && room, "null argument");
    GRB_REQUIRE(pool->timestamps && pool->page_table && pool->lengths && pool->overflow && pool->free_stack && pool->free_top &&
                    pool->errors && pool->row_of, "null pool pointer");
    GRB_REQUIRE(B > 0 && n > 0, "bad shape B=%d n=%d", B, n);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    HstuPoolArgs a = pool_args(pool, users, B);
    a.ids = reinterpret_cast<const long long*>(input_ids); a.n = n;
    a.room = room;
    launch_k(hstu_pool_alloc_kernel, 1, POOL_THREADS, 0, st, a);
    GRB_CUDA(cudaGetLastError());
    launch_k(hstu_cache_append_kernel, (unsigned)((B + 3) / 4), 128, 0, st, reinterpret_cast<const long long*>(input_ids),
             reinterpret_cast<const long long*>(timestamps), reinterpret_cast<const long long*>(users), (const int*)room, B, n,
             pool->max_items, KvPages{pool->page_table, pool_pt_ld(pool), pool->page_size}, reinterpret_cast<long long*>(pool->timestamps),
             pool->lengths, pool->overflow, positions, last_row);
    GRB_CUDA(cudaGetLastError());
    return 0;
}

int grb_hstu_pool_release(const grb_hstu_pool* pool, const int64_t* users, int B, float* last_hidden, int D, void* stream) {
    GRB_TRY(check_pool(pool));
    GRB_REQUIRE(users != nullptr, "null argument");
    GRB_REQUIRE(pool->page_table && pool->lengths && pool->overflow && pool->free_stack && pool->free_top && pool->errors && pool->row_of,
                "null pool pointer");
    GRB_REQUIRE(B > 0, "bad shape B=%d", B);
    GRB_REQUIRE(last_hidden == nullptr || D > 0, "last_hidden needs D > 0, got %d", D);
    HstuPoolArgs a = pool_args(pool, users, B);
    a.last_hidden = last_hidden; a.ld_hidden = D;
    launch_k(hstu_pool_release_kernel, 1, POOL_THREADS, 0, static_cast<cudaStream_t>(stream), a);
    GRB_CUDA(cudaGetLastError());
    return 0;
}

size_t grb_hstu_layer_extend_workspace_bytes(const grb_hstu_dims* d, int capacity) {
    if (check_extend(d, capacity)) return 0;
    return carve_extend(nullptr, d, capacity).bytes;
}

int grb_hstu_layer_extend(const grb_hstu_dims* d, const grb_hstu_layer_params* p, const grb_hstu_cache* c, int layer,
                          const int32_t* positions, const uint8_t* pos_bucket, int pos_bucket0, const int64_t* time_thr,
                          const float* x, float* y, void* workspace, void* stream) {
    GRB_REQUIRE(c != nullptr, "null cache");
    GRB_TRY(check_extend(d, c->capacity));
    GRB_REQUIRE(p && positions && x && y && workspace && c->kv && c->timestamps, "null argument");
    GRB_REQUIRE(c->B == d->B, "cache holds %d users, dims say B=%d", c->B, d->B);
    GRB_REQUIRE(layer >= 0 && layer < c->num_layers, "layer %d out of range [0, %d)", layer, c->num_layers);
    const int cap = c->capacity;
    ExtendKv kv{static_cast<bf16*>(c->kv) + (size_t)layer * d->B * cap * 2 * d->D, reinterpret_cast<const long long*>(c->timestamps),
                nullptr, KvPages{nullptr, 1, cap}, cap};
    return layer_extend(d, p, kv, positions, pos_bucket, pos_bucket0, time_thr, x, y, workspace, static_cast<cudaStream_t>(stream));
}

size_t grb_hstu_layer_extend_paged_workspace_bytes(const grb_hstu_dims* d, const grb_hstu_pool* pool) {
    if (check_pool(pool) || check_extend(d, pool->max_items)) return 0;
    return carve_extend(nullptr, d, pool->max_items).bytes;
}

int grb_hstu_layer_extend_paged(const grb_hstu_dims* d, const grb_hstu_layer_params* p, const grb_hstu_pool* pool, int layer,
                                const int64_t* users, const int32_t* positions, const uint8_t* pos_bucket, int pos_bucket0,
                                const int64_t* time_thr, const float* x, float* y, void* workspace, void* stream) {
    GRB_TRY(check_pool(pool));
    GRB_TRY(check_extend(d, pool->max_items));
    GRB_REQUIRE(p && users && positions && x && y && workspace && pool->kv && pool->timestamps && pool->page_table, "null argument");
    GRB_REQUIRE(layer >= 0 && layer < pool->num_layers, "layer %d out of range [0, %d)", layer, pool->num_layers);
    ExtendKv kv{static_cast<bf16*>(pool->kv) + (size_t)layer * pool->num_pages * pool->page_size * 2 * d->D,
                reinterpret_cast<const long long*>(pool->timestamps), reinterpret_cast<const long long*>(users),
                KvPages{pool->page_table, pool_pt_ld(pool), pool->page_size}, pool->max_items};
    return layer_extend(d, p, kv, positions, pos_bucket, pos_bucket0, time_thr, x, y, workspace, static_cast<cudaStream_t>(stream));
}

int grb_hstu_bias_index(const int64_t* timestamps, const uint8_t* pad, const int64_t* time_thr, const uint8_t* pos_bucket, int B, int L,
                        int npos, int ntime, uint16_t* out, int ld_index, void* stream) {
    GRB_REQUIRE(pad && time_thr && pos_bucket && out, "null argument");
    GRB_REQUIRE(B > 0 && L > 0 && B <= 65535 && L <= 65535, "bad shape B=%d L=%d", B, L);
    GRB_REQUIRE(ld_index >= L && ld_index % 8 == 0, "ld_index must be a multiple of 8 and >= L");
    GRB_REQUIRE(ntime >= 0 && ntime <= ATT_MAX_BUCKETS && npos >= 1 && npos <= ATT_MAX_BUCKETS, "bucket counts out of range");
    dim3 grid((ld_index + 255) / 256, (L + 7) / 8, B);
    auto go = [&](cudaStream_t s_) -> int {
        launch_k(hstu_bias_index_kernel, grid, 256, 0, s_, reinterpret_cast<const long long*>(timestamps), pad,
                 reinterpret_cast<const long long*>(time_thr), pos_bucket, L, ld_index, npos, ntime, out);
        GRB_CUDA(cudaGetLastError());
        return 0;
    };
    // the index matrix is first needed by the attention kernel of the first block: with the deferred schedule it is built beside
    // that block's cast + projection GEMM (grb_hstu_layer_forward joins before its attention launch)
    return run_maybe_deferred(static_cast<cudaStream_t>(stream), go);
}

int grb_set_defer_weight_grads(int on) {
    std::lock_guard<std::mutex> lock(g_defer_mu);
    g_defer_on = on != 0;
    return 0;
}
int grb_join_deferred(void* stream) { return join_pending(static_cast<cudaStream_t>(stream)); }

int grb_hstu_seq_prepare(const int64_t* timestamps, const uint8_t* pad, int B, int L, int32_t* rel32, uint8_t* wide, void* stream) {
    GRB_REQUIRE(timestamps && pad && rel32 && wide, "null argument");
    GRB_REQUIRE(B > 0 && L > 0, "bad shape B=%d L=%d", B, L);
    launch_k(hstu_seq_prep_kernel, (unsigned)B, 256, 0, static_cast<cudaStream_t>(stream), reinterpret_cast<const long long*>(timestamps), pad, L,
             reinterpret_cast<int*>(rel32), wide);
    GRB_CUDA(cudaGetLastError());
    return 0;
}

int grb_hstu_bucket_bytes_debug(const grb_hstu_seq* s, int B, int L, int ntime, uint8_t* out, void* stream) {
    GRB_REQUIRE(s && out && s->pad && s->time_thr, "null argument");
    GRB_REQUIRE(B > 0 && L > 0 && B <= 65535 && ntime >= 0 && ntime <= 64, "bad shape");
    HstuBucketArgs a;
    memset(&a, 0, sizeof(a));
    const bool has_time = s->timestamps != nullptr && s->has_time && ntime > 0;
    GRB_REQUIRE(!has_time || (s->rel32 && s->wide), "rel32 / wide missing: call grb_hstu_seq_prepare first");
    a.ts = has_time ? reinterpret_cast<const long long*>(s->timestamps) : nullptr;
    a.rel32 = s->rel32; a.wide = s->wide; a.pad = s->pad;
    a.thr64 = reinterpret_cast<const long long*>(s->time_thr);
    a.ntime = has_time ? ntime : 0;
    a.B = B; a.L = L;
    dim3 grid((L + 31) / 32, (L + 127) / 128, B);
    launch_k(hstu_bucket_bytes_debug_kernel, grid, 128, 0, static_cast<cudaStream_t>(stream), a, out);
    GRB_CUDA(cudaGetLastError());
    return 0;
}

size_t grb_hstu_attention_scratch_bytes(const grb_hstu_dims* d) {
    if (check_dims(d)) return 0;
    return align_up(attn_dw_part_floats(d->B, d->L, d->H) * sizeof(float));   // the bias-table gradient partials
}

int grb_hstu_attention_forward(const grb_hstu_dims* d, const float* pos_table, const float* time_table, const grb_hstu_seq* s,
                               const void* P_bf16, void* O_bf16, void* stream) {
    GRB_TRY(check_dims(d));
    GRB_REQUIRE(pos_table && P_bf16 && O_bf16, "null argument");
    GRB_TRY(check_seq(d, s));
    GRB_REQUIRE(aligned16(P_bf16) && aligned16(O_bf16), "buffers must be 16-byte aligned");
    HstuAttnArgs a = make_attn_args(d, pos_table, time_table, s, (const bf16*)P_bf16, (bf16*)O_bf16);
    return with_head_dim(d->D / d->H, [&](auto DH) { return launch_hstu_attn_fwd<DH>(a, static_cast<cudaStream_t>(stream)); });
}
int grb_hstu_attention_backward(const grb_hstu_dims* d, const float* pos_table, const float* time_table, const grb_hstu_seq* s,
                                const void* P_bf16, const void* zp_bf16, const void* dO_bf16, void* dzp_bf16, float* dpos_table,
                                float* dtime_table, void* scratch, void* stream) {
    GRB_TRY(check_dims(d));
    GRB_REQUIRE(pos_table && P_bf16 && dO_bf16 && dzp_bf16 && dpos_table && scratch, "null argument");
    GRB_TRY(check_seq(d, s));
    GRB_REQUIRE(aligned16(P_bf16) && aligned16(dO_bf16) && aligned16(dzp_bf16) && aligned16(scratch) && (zp_bf16 == nullptr || aligned16(zp_bf16)),
                "buffers must be 16-byte aligned");
    HstuAttnArgs a = make_attn_args(d, pos_table, time_table, s, (const bf16*)P_bf16, nullptr);
    GRB_TRY(set_attn_bwd_args(a, d, s, (const bf16*)dO_bf16, (const bf16*)zp_bf16, (bf16*)dzp_bf16, dpos_table, dtime_table,
                              static_cast<float*>(scratch)));
    return with_head_dim(d->D / d->H, [&](auto DH) { return launch_hstu_attn_bwd<DH>(a, static_cast<cudaStream_t>(stream)); });
}

int grb_collate_jagged(const int64_t* items, const int64_t* stamps, const int64_t* offsets, const int64_t* targets, int B, int L,
                       int64_t* out_input_ids, int64_t* out_targets, int64_t* out_timestamps, void* stream) {
    GRB_REQUIRE(items && offsets && targets && out_input_ids && out_targets, "null argument");
    GRB_REQUIRE(B > 0 && L > 0, "bad shape B=%d L=%d", B, L);
    const size_t n = (size_t)B * L;
    launch_k(collate_jagged_kernel, (unsigned)((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream), reinterpret_cast<const long long*>(items),
             reinterpret_cast<const long long*>(stamps), reinterpret_cast<const long long*>(offsets), reinterpret_cast<const long long*>(targets), B, L,
             reinterpret_cast<long long*>(out_input_ids), reinterpret_cast<long long*>(out_targets), reinterpret_cast<long long*>(out_timestamps));
    GRB_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------ embedding
int grb_embed_forward(const int64_t* ids, const float* table, const float* pos_table, float* x, uint8_t* pad, int B, int L, int D,
                      float scale, int mask_pad_rows, float dropout_p, uint64_t seed, const uint64_t* seed_dev, void* stream) {
    GRB_REQUIRE(ids && table && x, "null argument");
    GRB_REQUIRE(B > 0 && L > 0 && D > 0 && D % 4 == 0, "bad shape");
    EmbedArgs a{reinterpret_cast<const long long*>(ids), table, pos_table, x, pad, B * L, L, D, scale, mask_pad_rows,
                make_dropout(dropout_p, seed, SITE_EMBED, seed_dev)};
    launch_k(embed_fwd_kernel, row_grid(B * L), ROW_THREADS, 0, static_cast<cudaStream_t>(stream), a);
    GRB_CUDA(cudaGetLastError());
    return 0;
}
int grb_embed_backward(const int64_t* ids, const int64_t* order, const float* dx, float* dtable, float* dpos_table, int B, int L, int D,
                       float scale, int mask_pad_rows, float dropout_p, uint64_t seed, const uint64_t* seed_dev, float* scratch, void* stream) {
    GRB_REQUIRE(ids && order && dx && dtable && scratch, "null argument");
    GRB_REQUIRE(D <= 128 * EMB_MAX_CH, "embedding backward supports D <= %d", 128 * EMB_MAX_CH);
    GRB_REQUIRE(D % 4 == 0 && aligned16(dx) && aligned16(dtable) && aligned16(scratch) && (dpos_table == nullptr || aligned16(dpos_table)),
                "embedding backward needs D %% 4 == 0 and 16-byte aligned buffers");
    EmbedBwdArgs a{reinterpret_cast<const long long*>(ids), dx, dtable, dpos_table, B * L, L, D, scale, mask_pad_rows,
                   make_dropout(dropout_p, seed, SITE_EMBED, seed_dev), reinterpret_cast<const long long*>(order)};
    const EmbedPieceArgs pa{a, scratch};
    launch_k(embed_bwd_piece_kernel, row_grid((B * L + 31) / 32), ROW_THREADS, 0, static_cast<cudaStream_t>(stream), pa);
    GRB_CUDA(cudaGetLastError());
    launch_k(embed_bwd_run_kernel, row_grid(B * L), ROW_THREADS, 0, static_cast<cudaStream_t>(stream), pa);
    GRB_CUDA(cudaGetLastError());
    if (dpos_table) {
        launch_k(embed_bwd_kernel, row_grid(B * L), ROW_THREADS, 0, static_cast<cudaStream_t>(stream), a);
        GRB_CUDA(cudaGetLastError());
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------ head
namespace {
struct HeadWork {
    bf16* xf; float* stf; bf16* logits; float* dxf; float* scal;  // scal[0] = inv_count
    float* logits32;                                               // stored schedule: fp32 logits (the CE reads them, the bf16 buffer takes the gradient)
    float* row_loss;                                               // per-token loss, summed in a fixed order
    float* shift;                                                  // fused schedule: per-token log2-domain softmax shift
    float *part_ln, *part_tn;                                      // scratch of the ordered cross-CTA sums (LayerNorm, stored-schedule dE)
    int ldl;
    size_t bytes;
};
bool head_fused(int D) { return D <= 128; }
HeadWork carve_head(void* base, size_t T, size_t D, size_t C) {
    HeadWork h;
    Carver c{static_cast<char*>(base)};
    h.ldl = (int)((C + 7) / 8 * 8);
    h.xf = c.take<bf16>(T * D * 2);
    h.stf = c.take<float>(T * 2 * 4);
    h.dxf = c.take<float>(T * D * 4);
    h.scal = c.take<float>(64);
    // D <= 128: the fused kernels (tc_ce.cuh) never form the [T, C] logits; D = 256 stores them
    const bool fused = head_fused((int)D);
    h.logits = fused ? nullptr : c.take<bf16>(T * (size_t)h.ldl * 2);
    h.logits32 = fused ? nullptr : c.take<float>(T * (size_t)h.ldl * 4);
    h.row_loss = c.take<float>(T * 4);
    h.shift = c.take<float>(T * 4);
    h.part_ln = c.take<float>((size_t)2 * row_bwd_grid((int)T) * D * 4);
    const TnSpec spec{nullptr, nullptr, nullptr, (int)C, (int)D, (int)T, h.ldl, (int)D, (int)D};
    h.part_tn = fused ? nullptr : c.take<float>(tn_part_floats(&spec, 1, sm_count()) * 4);
    h.bytes = c.off;
    return h;
}
}  // namespace

size_t grb_head_workspace_bytes(int T, int D, int C) { return carve_head(nullptr, T, D, C).bytes; }

int grb_head_loss_forward_backward(const float* x, const float* ln_g, const float* ln_b, float ln_eps, const void* table_bf16,
                                   const int64_t* targets, int T, int D, int C, float* loss, float* dx, float* dtable, float* dln_g,
                                   float* dln_b, void* workspace, void* stream) {
    GRB_REQUIRE(x && ln_g && ln_b && table_bf16 && targets && loss && workspace, "null argument");
    GRB_REQUIRE(T > 0 && C > 1 && (D == 64 || D == 128 || D == 256), "bad shape T=%d D=%d C=%d", T, D, C);
    const bool want_grad = dx != nullptr;
    GRB_REQUIRE(!want_grad || (dtable && dln_g && dln_b), "null gradient pointer");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    HeadWork h = carve_head(workspace, T, D, C);
    // the target count (one CTA, latency-bound) depends on the targets only: with the deferred schedule it runs beside the final
    // LayerNorm and is joined before the CE kernel
    const bool count_aside = g_defer_on;
    auto count = [&](cudaStream_t s_) -> int {
        launch_k(ce_count_kernel, 1, 1024, 0, s_, reinterpret_cast<const long long*>(targets), T, h.scal, loss);
        GRB_CUDA(cudaGetLastError());
        return 0;
    };
    if (count_aside) GRB_TRY(defer_run(st, count));
    {
        LnFwdArgs a{x, ln_g, ln_b, h.xf, nullptr, h.stf, T, D, ln_eps};
        GRB_TRY(with_row_dim(D, [&](auto DC) { launch_k(ln_fwd_kernel<DC / 64>, row_grid(T), ROW_THREADS, 0, st, a); }));
    }
    if (count_aside) GRB_TRY(join_pending(st));
    else GRB_TRY(count(st));
    if (head_fused(D)) {
        // loss, dxf and the per-token shifts in one row-stationary pass; dE in a class-stationary pass (a weight gradient: off the
        // critical path with the deferred schedule)                                                      (hstu.py:137-146)
        CeArgs ca{reinterpret_cast<const long long*>(targets), h.scal, T, C, want_grad ? h.dxf : nullptr, h.shift, h.row_loss, dtable};
        if (D == 64) GRB_CUDA(launch_tc_ce<64>(h.xf, (const bf16*)table_bf16, ca, st));
        else GRB_CUDA(launch_tc_ce<128>(h.xf, (const bf16*)table_bf16, ca, st));
        launch_k(ce_loss_sum_kernel, 1, 1024, 0, st, (const float*)h.row_loss, T, loss);
        GRB_CUDA(cudaGetLastError());
        if (!want_grad) return 0;
        GRB_TRY(run_maybe_deferred(st, [&](cudaStream_t s_) -> int {
            if (D == 64) GRB_CUDA(launch_ce_table<64>(h.xf, (const bf16*)table_bf16, ca, s_));
            else GRB_CUDA(launch_ce_table<128>(h.xf, (const bf16*)table_bf16, ca, s_));
            return 0;
        }));
    } else {
    // logits = xf E^T   (hstu.py:137)
    GRB_CUDA((launch_tc_gemm<0>(h.xf, (const bf16*)table_bf16, T, C, D, D, D, TcEpiF32{nullptr, h.ldl, 1.f}, h.logits32, nullptr, h.ldl,
                                sm_count(), st)));
    if (h.ldl / 8 <= 256 * 8)
        launch_k(ce_fwd_bwd_vec_kernel<8>, T, 256, 0, st, h.logits, h.ldl, C, reinterpret_cast<const long long*>(targets), h.scal, h.row_loss, want_grad ? 1 : 0,
                 (const float*)h.logits32);
    else
        launch_k(ce_fwd_bwd_kernel, T, 256, 0, st, h.logits, h.ldl, C, reinterpret_cast<const long long*>(targets), h.scal, h.row_loss, want_grad ? 1 : 0,
                 (const float*)h.logits32);
    GRB_CUDA(cudaGetLastError());
    launch_k(ce_loss_sum_kernel, 1, 1024, 0, st, (const float*)h.row_loss, T, loss);
    GRB_CUDA(cudaGetLastError());
    if (!want_grad) return 0;
    GRB_CUDA(gemm_nn_f32(h.logits, (const bf16*)table_bf16, h.dxf, nullptr, 1.f, T, D, C, h.ldl, D, st));  // dxf = dlogits E
    // dE[C,D] += dlogits^T xf: a weight gradient, off the critical path with the deferred schedule
    TnSpec spec{h.logits, h.xf, dtable, C, D, T, h.ldl, D, D};
    GRB_TRY(run_maybe_deferred(st, [&](cudaStream_t s_) -> int {
        GRB_CUDA(launch_tc_tn_group(&spec, 1, sm_count(), h.part_tn, s_));
        return 0;
    }));
    }
    return ln_backward(LnBwdArgs{h.dxf, x, h.stf, ln_g, nullptr, dx, dln_g, dln_b, T, D, h.part_ln}, st);
}

int grb_head_logits(const float* x, const float* ln_g, const float* ln_b, float ln_eps, const void* table_bf16, int T, int D, int C,
                    float* logits, void* workspace, void* stream) {
    GRB_REQUIRE(x && ln_g && ln_b && table_bf16 && logits && workspace, "null argument");
    GRB_REQUIRE(T > 0 && C > 1 && (D == 64 || D == 128 || D == 256), "bad shape T=%d D=%d C=%d", T, D, C);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    HeadWork h = carve_head(workspace, T, D, C);
    {
        LnFwdArgs a{x, ln_g, ln_b, h.xf, nullptr, h.stf, T, D, ln_eps};
        GRB_TRY(with_row_dim(D, [&](auto DC) { launch_k(ln_fwd_kernel<DC / 64>, row_grid(T), ROW_THREADS, 0, st, a); }));
    }
    // logits [T, C] fp32, leading dimension C of any parity
    GRB_CUDA((launch_tc_gemm<0>(h.xf, (const bf16*)table_bf16, T, C, D, D, D, TcEpiF32Plain{logits, C}, nullptr, nullptr, 0, sm_count(), st)));
    return 0;
}

int grb_eval_rank_metrics(const float* logits, const int64_t* targets, int B, int C, float* metrics, int32_t* ranks, void* stream) {
    GRB_REQUIRE(logits && targets && metrics, "null argument");
    GRB_REQUIRE(B > 0 && C > 1, "bad shape B=%d C=%d", B, C);
    launch_k(eval_rank_kernel, (unsigned)B, 256, 0, static_cast<cudaStream_t>(stream), logits, C, reinterpret_cast<const long long*>(targets), metrics,
             reinterpret_cast<int*>(ranks));
    GRB_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------ SASRec attention
namespace {
int sas_args(const grb_sasrec_dims* d, SasAttnArgs& a) {
    GRB_REQUIRE(d && d->B > 0 && d->L > 0 && d->H > 0 && d->D % d->H == 0, "bad dims");
    int dh = d->D / d->H;
    GRB_REQUIRE(dh == 32 || dh == 64, "head_dim %d unsupported (32, 64)", dh);
    GRB_REQUIRE(d->D % 8 == 0, "embed_dim must be a multiple of 8");
    memset(&a, 0, sizeof(a));
    a.ld = d->D; a.B = d->B; a.L = d->L; a.H = d->H;
    a.scale = 1.f / sqrtf((float)dh);
    a.drop = make_dropout(d->dropout_p, d->seed, site_of(d->layer_index, SITE_ATTN), d->seed_dev);
    return 0;
}
}  // namespace

int grb_sasrec_attention_forward(const grb_sasrec_dims* d, const void* q, const void* k, const void* v, const uint8_t* pad, void* out,
                                 float* lse, void* stream) {
    SasAttnArgs a;
    GRB_TRY(sas_args(d, a));
    GRB_REQUIRE(q && k && v && pad && out && lse, "null argument");
    a.q = (const bf16*)q; a.k = (const bf16*)k; a.v = (const bf16*)v; a.pad = pad; a.out = (bf16*)out; a.lse = lse;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    dim3 grid((a.L + ATT_BLK - 1) / ATT_BLK, a.H, a.B);
    GRB_TRY(with_head_dim(d->D / d->H, [&](auto DH) -> int {
        GRB_TRY(set_smem(sas_attn_fwd_kernel<DH>, sizeof(SasSmem<DH>)));
        launch_k(sas_attn_fwd_kernel<DH>, grid, ATT_THREADS, sizeof(SasSmem<DH>), st, a);
        return 0;
    }));
    GRB_CUDA(cudaGetLastError());
    return 0;
}

int grb_sasrec_attention_backward(const grb_sasrec_dims* d, const void* q, const void* k, const void* v, const uint8_t* pad,
                                  const void* out, const float* lse, const void* dout, void* dq, void* dk, void* dv, void* stream) {
    SasAttnArgs a;
    GRB_TRY(sas_args(d, a));
    GRB_REQUIRE(q && k && v && pad && out && lse && dout && dq && dk && dv, "null argument");
    a.q = (const bf16*)q; a.k = (const bf16*)k; a.v = (const bf16*)v; a.pad = pad;
    a.out = (bf16*)const_cast<void*>(out); a.lse = const_cast<float*>(lse); a.d_out = (const bf16*)dout;
    a.dq = (bf16*)dq; a.dk = (bf16*)dk; a.dv = (bf16*)dv;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    dim3 grid((a.L + ATT_BLK - 1) / ATT_BLK, a.H, a.B);
    GRB_TRY(with_head_dim(d->D / d->H, [&](auto DH) -> int {
        GRB_TRY(set_smem(sas_attn_bwd_dq_kernel<DH>, sizeof(SasSmem<DH>)));
        GRB_TRY(set_smem(sas_attn_bwd_dkdv_kernel<DH>, sizeof(SasSmem<DH>)));
        launch_k(sas_attn_bwd_dq_kernel<DH>, grid, ATT_THREADS, sizeof(SasSmem<DH>), st, a);
        launch_k(sas_attn_bwd_dkdv_kernel<DH>, grid, ATT_THREADS, sizeof(SasSmem<DH>), st, a);
        return 0;
    }));
    GRB_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------ generic fused linear pieces
int grb_linear_forward(const void* x_bf16, const void* w_bf16, const float* bias, int T, int N, int K, int act, void* z_bf16,
                       void* act_bf16, float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t site, void* stream) {
    GRB_REQUIRE(x_bf16 && w_bf16 && bias && z_bf16, "null argument");
    GRB_REQUIRE(T > 0 && N % 8 == 0 && K % 8 == 0, "N and K must be multiples of 8");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Dropout drop = make_dropout(dropout_p, seed, site, seed_dev);
    GRB_REQUIRE(act >= 0 && act <= 2, "unknown activation %d", act);
    GRB_REQUIRE(act == 0 || act_bf16, "act output is null");
    GRB_CUDA(gemm_bias_act(act, (const bf16*)x_bf16, (const bf16*)w_bf16, bias, (bf16*)z_bf16, (bf16*)act_bf16, T, N, K, drop, st));
    return 0;
}
int grb_linear_residual_forward(const void* x_bf16, const void* w_bf16, const float* bias, const float* residual, const float* row_scale,
                                int T, int N, int K, float* y, float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t site,
                                void* stream) {
    GRB_REQUIRE(x_bf16 && w_bf16 && bias && residual && y, "null argument");
    GRB_REQUIRE(T > 0 && N % 8 == 0 && K % 8 == 0, "N and K must be multiples of 8");
    GRB_CUDA(gemm_bias_res((const bf16*)x_bf16, (const bf16*)w_bf16, bias, residual, row_scale, y, T, N, K,
                           make_dropout(dropout_p, seed, site, seed_dev), static_cast<cudaStream_t>(stream)));
    return 0;
}
namespace {
struct LinearBwdWork {
    float *part_colsum, *part_tn;
    size_t bytes;
};
// dW [N, K] += dy^T x: one problem of the grouped weight-gradient GEMM, dy [T, N] and x [T, K] stored token-major
TnSpec linear_dw_spec(const void* dy_bf16, const void* x_bf16, float* dw, int T, int N, int K) {
    return TnSpec{(const bf16*)dy_bf16, (const bf16*)x_bf16, dw, N, K, T, N, K, K};
}
LinearBwdWork carve_linear_bwd(void* base, int T, int N, int K) {
    LinearBwdWork w;
    Carver c{static_cast<char*>(base)};
    const dim3 cg = colsum_grid(T, N);
    w.part_colsum = c.take<float>((size_t)cg.x * cg.y * 256 * 4);
    const TnSpec spec = linear_dw_spec(nullptr, nullptr, nullptr, T, N, K);
    w.part_tn = c.take<float>(tn_part_floats(&spec, 1, sm_count()) * 4);
    w.bytes = c.off;
    return w;
}
}  // namespace

size_t grb_linear_backward_workspace_bytes(int T, int N, int K) {
    if (T <= 0 || N <= 0 || K <= 0) return 0;
    return carve_linear_bwd(nullptr, T, N, K).bytes;
}
int grb_linear_backward(const void* dy_bf16, const void* w_bf16, const void* x_bf16, int T, int N, int K, float* dx_f32,
                        const float* dx_residual, float* dw, float* db, void* workspace, void* stream) {
    GRB_REQUIRE(dy_bf16 && w_bf16, "null argument");
    GRB_REQUIRE(T > 0 && N % 8 == 0 && K % 8 == 0, "N and K must be multiples of 8");
    GRB_REQUIRE(workspace || (!dw && !db), "workspace is null");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const LinearBwdWork w = carve_linear_bwd(workspace, T, N, K);
    if (db) GRB_TRY(colsum((const bf16*)dy_bf16, T, N, N, db, w.part_colsum, st));
    if (dw) {
        GRB_REQUIRE(x_bf16, "x is null");
        const TnSpec spec = linear_dw_spec(dy_bf16, x_bf16, dw, T, N, K);
        GRB_CUDA(launch_tc_tn_group(&spec, 1, sm_count(), w.part_tn, st));
    }
    if (dx_f32) {
        GRB_CUDA(gemm_nn_f32((const bf16*)dy_bf16, (const bf16*)w_bf16, dx_f32, dx_residual, 1.f, T, K, N, N, K, st));
    }
    return 0;
}

int grb_linear_dact_backward(const void* dy_bf16, const void* w_bf16, const void* z_bf16, int T, int N, int K, int act, float dropout_p,
                             uint64_t seed, const uint64_t* seed_dev, uint32_t site, void* g_bf16, void* stream) {
    GRB_REQUIRE(dy_bf16 && w_bf16 && z_bf16 && g_bf16, "null argument");
    GRB_REQUIRE(T > 0 && N % 8 == 0 && K % 8 == 0 && (act == 1 || act == 2), "bad argument");
    GRB_CUDA(gemm_dact(act, (const bf16*)dy_bf16, (const bf16*)w_bf16, (const bf16*)z_bf16, (bf16*)g_bf16, T, K, N,
                       make_dropout(dropout_p, seed, site, seed_dev), static_cast<cudaStream_t>(stream)));
    return 0;
}
int grb_cast_rows_f32_to_bf16(const float* in, void* out_bf16, int T, int D, const float* row_scale, float dropout_p, uint64_t seed,
                              const uint64_t* seed_dev, uint32_t site, void* stream) {
    GRB_REQUIRE(in && out_bf16 && T > 0 && D > 0 && D % 4 == 0, "bad argument");
    return cast_bf16(in, (bf16*)out_bf16, (size_t)T * D, D, make_dropout(dropout_p, seed, site, seed_dev), row_scale,
                     static_cast<cudaStream_t>(stream));
}

int grb_layernorm_forward(const float* x, const float* g, const float* b, float eps, int T, int D, void* y_bf16, float* y_f32,
                          float* stats, void* stream) {
    GRB_REQUIRE(x && g && b && (y_bf16 || y_f32), "null argument");
    LnFwdArgs a{x, g, b, (bf16*)y_bf16, y_f32, stats, T, D, eps};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return with_row_dim(D, [&](auto DC) { launch_k(ln_fwd_kernel<DC / 64>, row_grid(T), ROW_THREADS, 0, st, a); });
}
size_t grb_layernorm_backward_workspace_bytes(int T, int D) {
    if (T <= 0 || D <= 0) return 0;
    return (size_t)2 * row_bwd_grid(T) * D * 4;
}
int grb_layernorm_backward(const float* dy, const float* x, const float* stats, const float* g, const float* residual, int T, int D,
                           float* dx, float* dg, float* db, void* workspace, void* stream) {
    GRB_REQUIRE(dy && x && stats && g && dx && dg && db && workspace, "null argument");
    return ln_backward(LnBwdArgs{dy, x, stats, g, residual, dx, dg, db, T, D, static_cast<float*>(workspace)}, static_cast<cudaStream_t>(stream));
}

int grb_split3_f32_to_bf16(const float* in, void* out_bf16, size_t rows, int K, int operand, void* stream) {
    GRB_REQUIRE(in && out_bf16 && K > 0 && (operand == 0 || operand == 1), "bad argument");
    if (rows == 0) return 0;
    launch_k(split3_f32_bf16_kernel, capped_blocks(rows * (size_t)K), 256, 0, static_cast<cudaStream_t>(stream), in, (bf16*)out_bf16, rows, K,
             operand);
    GRB_CUDA(cudaGetLastError());
    return 0;
}
static int linear_f32x3(const bf16* xs, const bf16* ws, const float* bias, const float* res2, int T, int N, int K, int act, float* y, int ldy,
                        cudaStream_t st) {
    const int K6 = 6 * K;
    // Two accumulators.  The tensor core adds each K = 16 group into the fp32 accumulator with truncation, an error relative to
    // the running sum per step: 288 steps over the six-term K (K = 768) measured 2e-5.  The five small cross terms (<= 2^-8 of
    // the result) are therefore summed on their own (their truncation is 2^-8 smaller), and the hi*hi term, K/16 steps, is
    // added to that sum in the epilogue of a second pass together with bias, activation and residual.  y doubles as the scratch of pass 1.
    GRB_CUDA((launch_tc_gemm<0>(xs + K, ws + K, T, N, 5 * K, K6, K6, TcEpiF32{nullptr, ldy, 1.f}, y, nullptr, ldy, sm_count(), st)));
    if (act == 1) GRB_CUDA((launch_tc_gemm<0>(xs, ws, T, N, K, K6, K6, TcEpiActResF32<1>{y, ldy, bias, res2}, y, nullptr, ldy, sm_count(), st)));
    else GRB_CUDA((launch_tc_gemm<0>(xs, ws, T, N, K, K6, K6, TcEpiActResF32<0>{y, ldy, bias, res2}, y, nullptr, ldy, sm_count(), st)));
    return 0;
}
int grb_linear_f32x3_forward(const void* x_split_bf16, const void* w_split_bf16, int T, int N, int K, int act, float* y, void* stream) {
    GRB_REQUIRE(x_split_bf16 && w_split_bf16 && y, "null argument");
    GRB_REQUIRE(T > 0 && N % 4 == 0 && K % 8 == 0 && (act == 0 || act == 1), "bad shape T=%d N=%d K=%d act=%d", T, N, K, act);
    GRB_REQUIRE(aligned16(x_split_bf16) && aligned16(w_split_bf16) && aligned16(y), "buffers must be 16-byte aligned");
    return linear_f32x3((const bf16*)x_split_bf16, (const bf16*)w_split_bf16, nullptr, nullptr, T, N, K, act, y, N, static_cast<cudaStream_t>(stream));
}
int grb_linear_f32x3_bias_forward(const void* x_split_bf16, const void* w_split_bf16, const float* bias, const float* residual, int T, int N,
                                  int K, int act, float* y, int ldy, void* stream) {
    GRB_REQUIRE(x_split_bf16 && w_split_bf16 && y, "null argument");
    GRB_REQUIRE(T > 0 && N > 0 && ldy >= N && ldy % 4 == 0 && K % 8 == 0 && (act == 0 || act == 1), "bad shape T=%d N=%d K=%d ldy=%d act=%d", T, N, K, ldy, act);
    GRB_REQUIRE(aligned16(x_split_bf16) && aligned16(w_split_bf16) && aligned16(y) && (!residual || aligned16(residual)), "buffers must be 16-byte aligned");
    return linear_f32x3((const bf16*)x_split_bf16, (const bf16*)w_split_bf16, bias, residual, T, N, K, act, y, ldy, static_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------------------------------------ fp32-exact HSTU block, forward
struct LayerF32Work {
    bf16* xs; float* P; float* O; float* x1; float* xn; float* h; bf16* hs; size_t bytes;
};
static LayerF32Work carve_f32(void* base, size_t T, size_t D) {
    LayerF32Work w;
    Carver c{static_cast<char*>(base)};
    w.xs = c.take<bf16>(T * 6 * D * 2);
    w.P = c.take<float>(T * 4 * D * 4);
    w.O = c.take<float>(T * D * 4);
    w.x1 = c.take<float>(T * D * 4);
    w.xn = c.take<float>(T * D * 4);
    w.h = c.take<float>(T * 4 * D * 4);
    w.hs = c.take<bf16>(T * 24 * D * 2);
    w.bytes = c.off;
    return w;
}
size_t grb_hstu_layer_f32_workspace_bytes(const grb_hstu_dims* d) {
    if (!d || d->B <= 0 || d->L <= 0 || d->D <= 0) return 0;
    return carve_f32(nullptr, (size_t)d->B * d->L, d->D).bytes;
}
int grb_hstu_layer_forward_f32(const grb_hstu_dims* d, const grb_hstu_layer_params_f32* p, const grb_hstu_seq* s, const float* x, float* y,
                               void* workspace, void* stream) {
    GRB_TRY(check_dims(d));
    GRB_REQUIRE(p && s && x && y && workspace, "null argument");
    GRB_REQUIRE(p->proj_w_split && p->proj_b && p->pos_table && p->ln1_g && p->ln1_b && p->ffn1_w_split && p->ffn1_b && p->ffn2_w_split &&
                    p->ffn2_b && p->ln2_g && p->ln2_b, "null parameter pointer");
    GRB_TRY(check_seq(d, s));
    GRB_REQUIRE(aligned16(x) && aligned16(y) && aligned16(workspace), "buffers must be 16-byte aligned");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int T = d->B * d->L, D = d->D;
    LayerF32Work w = carve_f32(workspace, T, D);
    GRB_TRY(join_pending(st));
    // P = silu(x Wp^T + bp)                                                                   (hstu.py:234-235)
    GRB_TRY(grb_split3_f32_to_bf16(x, w.xs, T, D, 0, stream));
    GRB_TRY(linear_f32x3(w.xs, (const bf16*)p->proj_w_split, p->proj_b, nullptr, T, 4 * D, D, 1, w.P, 4 * D, st));
    // O = silu(Q K^T + bias) V                                                                (hstu.py:244-267)
    {
        HstuAttnF32Args a{w.P, 4 * D, d->B, d->L, d->H, make_attn_bias(d, p->pos_table, p->time_table, s), w.O};
        GRB_REQUIRE(with_head_dim(D / d->H, [&](auto DH) { return launch_hstu_attn_f32<DH>(a, st); }) == 0, "fp32 attention launch failed");
    }
    // x1 = x + LN1(O) * U ; xn = LN2(x1)                                                      (hstu.py:271-278)
    {
        LnGateF32Args a{w.O, w.P, 4 * D, x, p->ln1_g, p->ln1_b, p->ln2_g, p->ln2_b, w.x1, w.xn, T, 1e-5f};
        GRB_TRY(with_row_dim(D, [&](auto DC) { launch_k(ln_gate_f32_kernel<DC / 32>, row_grid(T), 256, 0, st, a); }));
    }
    // y = x1 + (silu(xn W1^T + b1) W2^T + b2)                                                 (hstu.py:210-214, :278)
    GRB_TRY(grb_split3_f32_to_bf16(w.xn, w.xs, T, D, 0, stream));
    GRB_TRY(linear_f32x3(w.xs, (const bf16*)p->ffn1_w_split, p->ffn1_b, nullptr, T, 4 * D, D, 1, w.h, 4 * D, st));
    GRB_TRY(grb_split3_f32_to_bf16(w.h, w.hs, T, 4 * D, 0, stream));
    GRB_TRY(linear_f32x3(w.hs, (const bf16*)p->ffn2_w_split, p->ffn2_b, w.x1, T, D, 4 * D, 0, y, D, st));
    return 0;
}
int grb_layernorm_f32_forward(const float* x, const float* g, const float* b, float eps, int T, int D, float* y, void* stream) {
    GRB_REQUIRE(x && g && b && y && T > 0 && (D == 64 || D == 128 || D == 256), "bad argument T=%d D=%d", T, D);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return with_row_dim(D, [&](auto DC) { launch_k(ln_f32_kernel<DC / 32>, row_grid(T), 256, 0, st, x, g, b, y, T, eps); });
}

// ------------------------------------------------------------------------------------------------ T5-style attention core (TIGER)
static int t5_args(T5AttnArgs& a, const void* q, const void* k, const void* v, int B, int Lq, int Lk, int H, int DH, int ldq, int ldk, int ldv,
                   const float* bias, const int32_t* bucket, int nb, const uint8_t* key_pad, int causal, float scale, float p, uint64_t seed,
                   const uint64_t* seed_dev, uint32_t site) {
    GRB_REQUIRE(q && k && v, "null argument");
    GRB_REQUIRE(B > 0 && Lq > 0 && Lk > 0 && H > 0 && (DH == 32 || DH == 64), "bad shape B=%d Lq=%d Lk=%d H=%d head_dim=%d", B, Lq, Lk, H, DH);
    GRB_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && aligned16(q) && aligned16(k) && aligned16(v), "rows must be 16-byte aligned");
    GRB_REQUIRE((bias == nullptr) == (bucket == nullptr) && (!bias || (nb > 0 && nb <= 1024)), "bias table and bucket map go together");
    GRB_REQUIRE(p >= 0.f && p < 1.f, "dropout_p out of range");
    memset(&a, 0, sizeof(a));
    a.q = (const bf16*)q; a.k = (const bf16*)k; a.v = (const bf16*)v; a.ldq = ldq; a.ldk = ldk; a.ldv = ldv;
    a.B = B; a.Lq = Lq; a.Lk = Lk; a.H = H; a.bias = bias; a.bucket = bucket; a.nb = bias ? nb : 0; a.key_pad = key_pad; a.causal = causal;
    a.scale = scale; a.drop = make_dropout(p, seed, site, seed_dev);
    return 0;
}
int grb_t5_attention_forward(const void* q, const void* k, const void* v, int B, int Lq, int Lk, int H, int head_dim, int ldq, int ldk, int ldv,
                             const float* bias, const int32_t* bucket, int num_buckets, const uint8_t* key_pad, int causal, float scale,
                             float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t site, void* out, int ldo, float* lse,
                             void* stream) {
    T5AttnArgs a;
    GRB_TRY(t5_args(a, q, k, v, B, Lq, Lk, H, head_dim, ldq, ldk, ldv, bias, bucket, num_buckets, key_pad, causal, scale, dropout_p, seed, seed_dev, site));
    GRB_REQUIRE(out && lse && ldo % 8 == 0 && aligned16(out), "bad output");
    a.out = (bf16*)out; a.ldo = ldo; a.lse = lse;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    dim3 grid((Lq + T5_ROWS - 1) / T5_ROWS, B * H);
    GRB_TRY(with_head_dim(head_dim, [&](auto DH) -> int {
        const size_t smem = t5_fwd_smem<DH>(a.nb);
        GRB_TRY(set_smem(t5_attn_fwd_kernel<DH>, smem));
        launch_k(t5_attn_fwd_kernel<DH>, grid, T5_THREADS, smem, st, a);
        return 0;
    }));
    GRB_CUDA(cudaGetLastError());
    return 0;
}
int grb_t5_attention_backward(const void* q, const void* k, const void* v, int B, int Lq, int Lk, int H, int head_dim, int ldq, int ldk, int ldv,
                              const float* bias, const int32_t* bucket, int num_buckets, const uint8_t* key_pad, int causal, float scale,
                              float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t site, const void* out, int ldo,
                              const float* lse, const void* dout, int lddo, void* dq, int lddq, float* dk, float* dv, float* dbias,
                              void* stream) {
    T5AttnArgs a;
    GRB_TRY(t5_args(a, q, k, v, B, Lq, Lk, H, head_dim, ldq, ldk, ldv, bias, bucket, num_buckets, key_pad, causal, scale, dropout_p, seed, seed_dev, site));
    GRB_REQUIRE(out && lse && dout && dq && dk && dv && ldo % 8 == 0 && lddo % 8 == 0 && lddq % 8 == 0, "bad argument");
    GRB_REQUIRE(aligned16(out) && aligned16(dout) && aligned16(dq), "rows must be 16-byte aligned");
    a.out = (bf16*)const_cast<void*>(out); a.ldo = ldo; a.lse = const_cast<float*>(lse); a.dout = (const bf16*)dout; a.lddo = lddo;
    a.dq = (bf16*)dq; a.lddq = lddq; a.dk = dk; a.dv = dv; a.dbias = bias ? dbias : nullptr;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    GRB_CUDA(cudaMemsetAsync(dk, 0, (size_t)B * Lk * H * head_dim * sizeof(float), st));
    GRB_CUDA(cudaMemsetAsync(dv, 0, (size_t)B * Lk * H * head_dim * sizeof(float), st));
    dim3 grid((Lq + T5_ROWS - 1) / T5_ROWS, B * H);
    GRB_TRY(with_head_dim(head_dim, [&](auto DH) -> int {
        const size_t smem = t5_bwd_smem<DH>(a.nb);
        GRB_TRY(set_smem(t5_attn_bwd_kernel<DH>, smem));
        launch_k(t5_attn_bwd_kernel<DH>, grid, T5_THREADS, smem, st, a);
        return 0;
    }));
    GRB_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------ TIGER constrained beam step
int grb_trie_log_softmax(const float* logits, int rows, int V, const int32_t* node, const int32_t* child_off, const int32_t* child_tok,
                         int n_nodes, int use_trie, int vocab_offset, int num_embeddings, float temperature, float* probs, float* logp,
                         void* stream) {
    GRB_REQUIRE(logits && probs && logp && rows >= 0 && V > 0 && V <= 1 << 20, "bad argument rows=%d V=%d", rows, V);
    GRB_REQUIRE(!use_trie || (node && child_off && n_nodes > 0), "trie arrays missing");
    GRB_REQUIRE(temperature > 0.f, "temperature must be positive");
    if (rows == 0) return 0;
    TrieCsr t{child_off, child_tok, nullptr, n_nodes};
    const size_t smem = (size_t)((V + 31) / 32) * 4;
    launch_k(trie_log_softmax_kernel, rows, 256, smem, static_cast<cudaStream_t>(stream), logits, V, node, t, use_trie, vocab_offset,
             num_embeddings, temperature, probs, logp);
    GRB_CUDA(cudaGetLastError());
    return 0;
}
int grb_beam_select(const int64_t* beam_seqs, const float* beam_logps, const int64_t* cand_tok, const float* cand_logp, const int32_t* nodes,
                    const int32_t* child_off, const int32_t* child_tok, const int32_t* child_node, int n_nodes, int B, int K, int KK, int S,
                    int64_t* new_seqs, float* new_logps, int32_t* new_nodes, void* stream) {
    GRB_REQUIRE(beam_logps && cand_tok && cand_logp && new_seqs && new_logps && (S == 0 || beam_seqs), "null argument");
    GRB_REQUIRE(B >= 0 && K >= 1 && K <= 32 && KK >= 1 && K * KK <= BEAM_MAX_CAND && S >= 0, "bad shape B=%d K=%d KK=%d S=%d (K <= 32, K*KK <= 1024)", B, K, KK, S);
    GRB_REQUIRE(!new_nodes || (nodes && child_off && child_tok && child_node && n_nodes > 0), "trie arrays missing");
    if (B == 0) return 0;
    BeamSelectArgs a{reinterpret_cast<const long long*>(beam_seqs), beam_logps, reinterpret_cast<const long long*>(cand_tok), cand_logp, nodes,
                     TrieCsr{child_off, child_tok, child_node, n_nodes}, K, KK, S, reinterpret_cast<long long*>(new_seqs), new_logps, new_nodes};
    launch_k(beam_select_kernel, B, BEAM_MAX_CAND, 0, static_cast<cudaStream_t>(stream), a);
    GRB_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------ optimizer / casts
int grb_cast_f32_to_bf16(const float* in, void* out_bf16, size_t n, void* stream) {
    GRB_REQUIRE(in && out_bf16, "null argument");
    if (n == 0) return 0;
    launch_k(cast_flat_f32_bf16_kernel, capped_blocks(n), 256, 0, static_cast<cudaStream_t>(stream), in, (bf16*)out_bf16, n);
    GRB_CUDA(cudaGetLastError());
    return 0;
}
int grb_adam_step(float* p, float* g, float* m, float* v, void* p_bf16, size_t n, float* state, float lr, float beta1, float beta2,
                  float eps, float weight_decay, float grad_scale, int zero_grad, void* stream) {
    GRB_REQUIRE(p && g && m && v && state, "null argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    launch_k(adam_tick_kernel, 1, 1, 0, st, state, beta1, beta2);
    GRB_CUDA(cudaGetLastError());
    if (n == 0) return 0;
    AdamArgs a{p, g, m, v, (bf16*)p_bf16, n, state, lr, beta1, beta2, eps, weight_decay, grad_scale, zero_grad};
    launch_k(adam_step_kernel, capped_blocks(n), 256, 0, st, a);
    GRB_CUDA(cudaGetLastError());
    return 0;
}

int grb_dp_adam_step(float* p, float* g, float* m, float* v, void* p_bf16, const void* mc_g, void* mc_p, void* mc_p_bf16,
                     const void* peer_g, const void* peer_p, const void* peer_p_bf16, const void* peer_sig, void* sig, void* epoch,
                     size_t n, int rank, int world, float* state, float lr, float beta1, float beta2, float eps, float weight_decay,
                     float grad_scale, void* stream) {
    GRB_REQUIRE(p && g && m && v && p_bf16 && peer_sig && sig && epoch && state, "null argument");
    GRB_REQUIRE(world >= 2 && world <= 32 && rank >= 0 && rank < world, "bad rank/world %d/%d", rank, world);
    GRB_REQUIRE(n > 0 && n % ((size_t)8 * world) == 0, "n must be a multiple of 8 * world");
    const bool mc = mc_g != nullptr && mc_p != nullptr && mc_p_bf16 != nullptr;
    GRB_REQUIRE(mc || (peer_g && peer_p && peer_p_bf16), "neither multicast addresses nor peer pointer arrays given");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    launch_k(adam_tick_kernel, 1, 1, 0, st, state, beta1, beta2);
    GRB_CUDA(cudaGetLastError());
    launch_k(dp_barrier_kernel, 1, 32, 0, st, reinterpret_cast<unsigned* const*>(peer_sig), reinterpret_cast<unsigned*>(sig),
             reinterpret_cast<unsigned*>(epoch), rank, world, 0);
    GRB_CUDA(cudaGetLastError());
    DpAdamArgs a{p, g, m, v, (bf16*)p_bf16, (const float*)mc_g, (float*)mc_p, (bf16*)mc_p_bf16,
                 reinterpret_cast<const float* const*>(peer_g), reinterpret_cast<float* const*>(peer_p), reinterpret_cast<bf16* const*>(peer_p_bf16),
                 n, rank, world, state, lr, beta1, beta2, eps, weight_decay, grad_scale};
    const unsigned blocks = capped_blocks(n / world / 8, 4);
    if (mc) launch_k(dp_adam_kernel<true>, blocks, 256, 0, st, a);
    else launch_k(dp_adam_kernel<false>, blocks, 256, 0, st, a);
    GRB_CUDA(cudaGetLastError());
    launch_k(dp_barrier_kernel, 1, 32, 0, st, reinterpret_cast<unsigned* const*>(peer_sig), reinterpret_cast<unsigned*>(sig),
             reinterpret_cast<unsigned*>(epoch), rank, world, 1);
    GRB_CUDA(cudaGetLastError());
    GRB_CUDA(cudaMemsetAsync(g, 0, n * sizeof(float), st));
    return 0;
}

namespace {
__global__ void assert_unit_scalar_kernel(const float* v) {
    pdl_wait();
    if (*v != 1.0f) {
        printf("genrec_b200: the loss was back-propagated with gradient %g, but FlatAdam(unit_loss_grad=True) promised 1\n", (double)*v);
        __trap();
    }
}
}  // namespace
int grb_assert_unit_scalar(const float* value, void* stream) {
    GRB_REQUIRE(value, "null argument");
    launch_k(assert_unit_scalar_kernel, 1, 1, 0, static_cast<cudaStream_t>(stream), value);
    GRB_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------ RQ-VAE
int grb_rq_residual_argmin(const float* x, const float* codebooks, int64_t N, int D, int K, int levels, float commitment, int64_t* ids,
                           float* emb, float* res, float* loss, float* res_out, void* stream) {
    GRB_REQUIRE(x && codebooks && ids, "null argument");
    GRB_REQUIRE(N >= 0 && levels >= 1 && K >= 2 && K % 2 == 0, "bad shape N=%lld K=%d levels=%d", (long long)N, K, levels);
    GRB_REQUIRE(D == 32 || D == 64, "latent dim %d unsupported (32, 64)", D);
    GRB_REQUIRE((size_t)K * (D + 1) * 4 <= 200 * 1024, "codebook level does not fit shared memory (K=%d, D=%d)", K, D);
    GRB_REQUIRE(aligned16(x) && aligned16(codebooks), "buffers must be 16-byte aligned");
    if (N == 0) return 0;
    RqArgs a{x, codebooks, reinterpret_cast<long long*>(ids), emb, res, loss, res_out, (long long)N, K, levels, commitment};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    GRB_REQUIRE(emb == nullptr || aligned16(emb), "emb must be 16-byte aligned");
    GRB_REQUIRE(res == nullptr || aligned16(res), "res must be 16-byte aligned");
    // Three kernels (rq_argmin.cuh).  Default: the register-blocked tile kernel (D = 32, K a multiple of 256, tile fits shared
    // memory).  GRB_RQ = tile | split | thread forces one; split / thread are the earlier generations, kept as cross-checks
    // (tests/test_rq_gpu.py compares all three) and for the shapes the tile kernel does not cover.
    const char* rq_env = getenv("GRB_RQ");
    const bool force_thread = rq_env != nullptr && strcmp(rq_env, "thread") == 0;
    const bool force_split = rq_env != nullptr && strcmp(rq_env, "split") == 0;
    {
        const bool stage = emb != nullptr || res != nullptr;
        const size_t smem = rq_tile_smem_bytes(D, K, levels, stage);
        if (!force_thread && !force_split && D == 32 && K % 256 == 0 && smem <= 220 * 1024) {
            GRB_TRY(set_smem(rq_residual_argmin_tile_kernel<32>, smem));
            const unsigned grid = (unsigned)((N + RQT_ROWS - 1) / RQT_ROWS);
            launch_k(rq_residual_argmin_tile_kernel<32>, grid, RQT_THREADS, smem, st, a);
            GRB_CUDA(cudaGetLastError());
            return 0;
        }
    }
    const bool legacy = force_thread || (!force_split && N > (int64_t)sm_count() * RQ_THREADS * 4);
    if (!legacy && K % 8 == 0) {
        // four threads per row (see rq_argmin.cuh); two rows per thread once there is more than a wave of work (FMA : LDS = 8 : 1)
        const int rows = (D == 32 && N > (int64_t)sm_count() * RQ_ROWS_PER_CTA * 4) ? 2 : 1;
        const size_t base = ((size_t)K * D + ((K + 3) & ~3)) * sizeof(float);
        const size_t stage = (emb || res) ? (size_t)2 * RQ_ROWS_PER_CTA * rows * D * levels * sizeof(float) : 0;
        const bool staged = stage > 0 && base + stage <= 200 * 1024;
        const size_t smem = base + (staged ? stage : 0);
        const unsigned grid = (unsigned)((N + (int64_t)RQ_ROWS_PER_CTA * rows - 1) / ((int64_t)RQ_ROWS_PER_CTA * rows));
        auto go = [&](auto kern) -> int {
            GRB_TRY(set_smem(kern, smem));
            launch_k(kern, grid, RQ_THREADS, smem, st, a);
            return 0;
        };
        if (D == 32) {
            if (rows == 2) GRB_TRY(staged ? go(rq_residual_argmin_split_kernel<32, 2, true>) : go(rq_residual_argmin_split_kernel<32, 2, false>));
            else GRB_TRY(staged ? go(rq_residual_argmin_split_kernel<32, 1, true>) : go(rq_residual_argmin_split_kernel<32, 1, false>));
        } else {
            GRB_TRY(staged ? go(rq_residual_argmin_split_kernel<64, 1, true>) : go(rq_residual_argmin_split_kernel<64, 1, false>));
        }
        GRB_CUDA(cudaGetLastError());
        return 0;
    }
    size_t smem = (size_t)K * (D + 1) * sizeof(float);
    if (D == 32) {
        // two rows per thread once there is more than a wave of work; one row per thread for small N (more CTAs)
        if (N > (int64_t)sm_count() * RQ_THREADS * 2) {
            unsigned grid = (unsigned)((N + 2 * RQ_THREADS - 1) / (2 * RQ_THREADS));
            GRB_TRY(set_smem(rq_residual_argmin_kernel<32, 2>, smem));
            launch_k(rq_residual_argmin_kernel<32, 2>, grid, RQ_THREADS, smem, st, a);
        } else {
            unsigned grid = (unsigned)((N + RQ_THREADS - 1) / RQ_THREADS);
            GRB_TRY(set_smem(rq_residual_argmin_kernel<32, 1>, smem));
            launch_k(rq_residual_argmin_kernel<32, 1>, grid, RQ_THREADS, smem, st, a);
        }
    } else {
        unsigned grid = (unsigned)((N + RQ_THREADS - 1) / RQ_THREADS);
        GRB_TRY(set_smem(rq_residual_argmin_kernel<64, 1>, smem));
        launch_k(rq_residual_argmin_kernel<64, 1>, grid, RQ_THREADS, smem, st, a);
    }
    GRB_CUDA(cudaGetLastError());
    return 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ RQ-VAE training: Sinkhorn, k-means
namespace {
size_t sk_workspace(int64_t B, int K) {
    return align_up((size_t)B * sizeof(double)) + (sk_kmat_in_smem(B, K) ? 0 : align_up((size_t)B * K * sizeof(double)));
}
// once per device: both instantiations may use the full opt-in shared memory and the non-portable cluster size, and one cluster of
// SK_CLUSTER such CTAs must fit the device
int sk_prepare() {
    static std::mutex mu;
    static bool ready[64] = {false};
    std::lock_guard<std::mutex> lock(mu);
    const int dev = current_device() & 63;
    if (ready[dev]) return 0;
    for (auto kern : {rq_sinkhorn_kernel<true>, rq_sinkhorn_kernel<false>}) {
        GRB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
        GRB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SK_SMEM_MAX));
        cudaLaunchConfig_t cfg;
        memset(&cfg, 0, sizeof(cfg));
        cfg.gridDim = dim3(SK_CLUSTER);
        cfg.blockDim = dim3(SK_THREADS);
        cfg.dynamicSmemBytes = SK_SMEM_MAX;
        cudaLaunchAttribute at;
        at.id = cudaLaunchAttributeClusterDimension;
        at.val.clusterDim.x = SK_CLUSTER;
        at.val.clusterDim.y = 1;
        at.val.clusterDim.z = 1;
        cfg.attrs = &at;
        cfg.numAttrs = 1;
        int n = 0;
        GRB_CUDA(cudaOccupancyMaxActiveClusters(&n, kern, &cfg));
        if (n < 1) return fail(GRB_ENODEV, "rq_sinkhorn: a cluster of %d CTAs x %d threads with %zu B of shared memory does not fit this device",
                               SK_CLUSTER, SK_THREADS, SK_SMEM_MAX);
    }
    ready[dev] = true;
    return 0;
}
}  // namespace

extern "C" {

size_t grb_rq_sinkhorn_workspace_bytes(int64_t B, int K) {
    if (B < 0 || K < 2 || K > SK_KMAX) {
        fail(GRB_EINVAL, "rq_sinkhorn: B=%lld K=%d unsupported (B >= 0, 2 <= K <= %d)", (long long)B, K, SK_KMAX);
        return 0;
    }
    return sk_workspace(B, K);
}

int grb_rq_sinkhorn(const float* dist, int64_t B, int K, double eps, int iters, int64_t* ids, double* u_out, double* v_out,
                    void* workspace, void* stream) {
    GRB_REQUIRE(B >= 0 && K >= 2 && K <= SK_KMAX, "rq_sinkhorn: B=%lld K=%d unsupported (B >= 0, 2 <= K <= %d)", (long long)B, K, SK_KMAX);
    GRB_REQUIRE(iters >= 0 && eps > 0.0 && eps < INFINITY, "rq_sinkhorn: iters=%d eps=%g unsupported (iters >= 0, eps > 0 finite)", iters, eps);
    if (B == 0) return 0;
    GRB_REQUIRE(dist && ids && workspace, "rq_sinkhorn: null argument (dist, ids and workspace are required)");
    GRB_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 7) == 0, "rq_sinkhorn: workspace must be 8-byte aligned");
    GRB_TRY(sk_prepare());
    const bool in_smem = sk_kmat_in_smem(B, K);
    const size_t rows = sk_rows_per_cta(B);
    double* u = static_cast<double*>(workspace);
    double* kmat = in_smem ? nullptr : reinterpret_cast<double*>(static_cast<char*>(workspace) + align_up((size_t)B * sizeof(double)));
    SinkhornArgs a{dist, (long long)B, K, iters, (int)rows, eps, reinterpret_cast<long long*>(ids), u_out, v_out, u, kmat};
    const size_t smem = SK_SMEM_FIXED + (in_smem ? rows * K * sizeof(double) : 0);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (in_smem) launch_kc(rq_sinkhorn_kernel<true>, SK_CLUSTER, SK_THREADS, SK_CLUSTER, smem, st, a);
    else launch_kc(rq_sinkhorn_kernel<false>, SK_CLUSTER, SK_THREADS, SK_CLUSTER, smem, st, a);
    GRB_CUDA(cudaGetLastError());
    return 0;
}

int grb_kmeans_update(const float* x, const int64_t* assign, int64_t B, int D, int k, float* centroids, int32_t* counts, float* shift,
                      void* stream) {
    GRB_REQUIRE(B >= 0 && k >= 1 && k <= (1 << 20) && D >= 1 && D <= KM_THREADS,
                "kmeans_update: B=%lld D=%d k=%d unsupported (B >= 0, 1 <= D <= %d, 1 <= k <= 2^20)", (long long)B, D, k, KM_THREADS);
    GRB_REQUIRE(x && assign && centroids && counts && shift, "kmeans_update: null argument");
    launch_k(kmeans_update_kernel, (unsigned)k, KM_THREADS, 0, static_cast<cudaStream_t>(stream), x, reinterpret_cast<const long long*>(assign),
             (long long)B, D, centroids, counts, shift);
    GRB_CUDA(cudaGetLastError());
    return 0;
}

}  // extern "C"
