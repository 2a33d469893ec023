// genrec_b200 - lazy Adam for one table of the flat buffer: only the rows a step touched are updated (FlatAdam(lazy_table=True)).
//
// The table's gradient slot stays a dense [C, D] block of the flat gradient; what becomes proportional to the touched rows is the
// per-step work over it.  A row set lives in three device buffers: flag [C] int32, rows [C] int32 and count, plus an "all" word.
//   rowset_mark_kernel      flag[id] = 1 for every id in 1 .. C-1 of an id vector; the thread that flips a flag appends its id to
//                           rows (atomicCAS on the flag, one atomicAdd on count per warp).  O(ids), never O(C); the list cannot
//                           overflow (capacity C).  Its order depends on timing; the step's result does not, as every row is
//                           updated on its own.
//   rowset_mark_all_kernel  all = 1: the next step walks every row 0 .. C-1 (the full softmax head writes into all of them).
//   lazy_table_step_kernel  a fixed grid walks rows[0 .. count), or every row when all is set: adam_update (the dense kernel's
//                           per-element function) on p, m, v, the bf16 mirror, the gradient row zeroed, flag[row] cleared.
//                           float4 accesses (8 bytes of mirror).
//   rowset_reset_kernel     count = all = 0, launched after the step, once every CTA has read them.
// Everything reads its sizes on the device, so a captured step follows whatever rows the replayed forwards mark.
#pragma once
#include "rowwise.cuh"

namespace grb {

__global__ void __launch_bounds__(256) rowset_mark_kernel(const long long* __restrict__ ids, size_t n, int C, int* __restrict__ flag,
                                                          int* __restrict__ rows, int* __restrict__ count) {
    pdl_wait();
    const int lane = threadIdx.x & 31;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    // the loop bound is tested on the warp's first index, so every lane of a warp runs the same iterations (ballot below)
    for (size_t i0 = (size_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31); i0 < n; i0 += stride) {
        const size_t i = i0 + lane;
        int id = 0;
        bool fresh = false;
        if (i < n) {
            const long long x = ids[i];
            if (x >= 1 && x < C) {
                id = (int)x;
                fresh = flag[id] == 0 && atomicCAS(flag + id, 0, 1) == 0;
            }
        }
        const unsigned b = __ballot_sync(0xffffffffu, fresh);
        if (b == 0u) continue;
        const int leader = __ffs(b) - 1;
        int base = 0;
        if (lane == leader) base = atomicAdd(count, __popc(b));
        base = __shfl_sync(0xffffffffu, base, leader);
        if (fresh) rows[base + __popc(b & ((1u << lane) - 1u))] = id;
    }
}

__global__ void rowset_mark_all_kernel(int* all) {
    pdl_wait();
    *all = 1;
}

__global__ void rowset_reset_kernel(int* count, int* all) {
    pdl_wait();
    *count = 0;
    *all = 0;
}

struct LazyTableArgs {
    float* p; float* g; float* m; float* v; bf16* p_bf16;   // the table's slot of each flat buffer, [C, D]
    int C;
    int* flag;
    const int* rows;
    const int* count;
    const int* all;
    const float* state;
    float lr, beta1, beta2, eps, weight_decay, grad_scale;
};

// D4 = D / 4 float4 columns per row; one thread per (listed row, float4 column), grid-stride
template <int D4>
__global__ void __launch_bounds__(256) lazy_table_step_kernel(LazyTableArgs a) {
    pdl_wait();
    const float bc1 = a.state[1], bc2 = a.state[2];
    const float step_size = a.lr / bc1;
    const float inv_sqrt_bc2 = rsqrtf(bc2);
    const bool all = *a.all != 0;
    const size_t total = (all ? (size_t)a.C : (size_t)*a.count) * D4;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride) {
        const size_t r = e / D4;
        const int c = (int)(e % D4);
        const size_t row = all ? r : (size_t)a.rows[r];
        const size_t o = row * (4 * D4) + 4 * c;
        float4 p = *reinterpret_cast<const float4*>(a.p + o);
        const float4 g = *reinterpret_cast<const float4*>(a.g + o);
        float4 m = *reinterpret_cast<const float4*>(a.m + o);
        float4 v = *reinterpret_cast<const float4*>(a.v + o);
        p.x = adam_update(p.x, g.x, m.x, v.x, a.grad_scale, a.beta1, a.beta2, a.eps, a.weight_decay, step_size, inv_sqrt_bc2);
        p.y = adam_update(p.y, g.y, m.y, v.y, a.grad_scale, a.beta1, a.beta2, a.eps, a.weight_decay, step_size, inv_sqrt_bc2);
        p.z = adam_update(p.z, g.z, m.z, v.z, a.grad_scale, a.beta1, a.beta2, a.eps, a.weight_decay, step_size, inv_sqrt_bc2);
        p.w = adam_update(p.w, g.w, m.w, v.w, a.grad_scale, a.beta1, a.beta2, a.eps, a.weight_decay, step_size, inv_sqrt_bc2);
        *reinterpret_cast<float4*>(a.p + o) = p;
        *reinterpret_cast<float4*>(a.m + o) = m;
        *reinterpret_cast<float4*>(a.v + o) = v;
        *reinterpret_cast<float4*>(a.g + o) = make_float4(0.f, 0.f, 0.f, 0.f);
        *reinterpret_cast<uint2*>(a.p_bf16 + o) = make_uint2(pack_bf16(p.x, p.y), pack_bf16(p.z, p.w));
        if (c == 0) a.flag[row] = 0;
    }
}

}  // namespace grb
