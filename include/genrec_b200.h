/* genrec_b200 - C ABI of the H100-native (sm_90a) hot path of phonism/genrec.
 *
 * The reference is pure Python/PyTorch: it has no FFI of its own.  The interface each entry point below replaces is
 * therefore the body of the reference nn.Module method named in its comment (file:line under /root/reference); the
 * reference-side binding a maintainer adds is the ctypes stub shown in INTEGRATION.md (and shipped as
 * genrec_b200/_lib.py).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the parameter name ends in _host; no torch types cross this boundary;
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, nothing synchronises, nothing allocates:
 *     scratch and saved-for-backward storage is caller-provided (sizes from the *_bytes() queries), so every entry
 *     point is CUDA-graph capturable;
 *   - return value 0 = success; otherwise a negative GRB_E* code, text via grb_last_error();
 *   - activations: T = B*L token rows, row-major [T, D]; fp32 residual stream, bf16 tensor-core operands;
 *   - "bf16" pointers are void* to 2-byte bfloat16 storage;
 *   - gradient outputs of parameters are ACCUMULATED (+=) so they can point straight into a flat, pre-zeroed grad buffer.
 */
#ifndef GENREC_B200_H
#define GENREC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GRB_OK 0
#define GRB_EINVAL (-1)   /* unsupported shape / null pointer / misaligned buffer */
#define GRB_ECUDA (-2)    /* a CUDA launch or runtime call failed */
#define GRB_ENODEV (-3)   /* no sm_90 device */

const char* grb_last_error(void);
int grb_version(void);
/* number of CUDA kernels this library has launched in this process so far (host-side count at launch / graph-capture time) */
uint64_t grb_launch_count(void);
/* 0 when device `ordinal` is compute capability 10.x, GRB_ENODEV otherwise (host call). */
int grb_check_device(int ordinal);

/* ------------------------------------------------------------------------------------------------ HSTU block
 * Replaces HSTULayer.forward (genrec/models/hstu.py:222-280) incl. RelativePositionBias.forward (:330-349) and
 * TemporalBias.forward (:386-409), and their autograd backward. */
typedef struct {
    int B, L, D, H;          /* head_dim = D / H must be 32 or 64 ; D in {64,128,256} */
    int npos, ntime;         /* bucket counts of the two bias tables, each <= 64 ; ntime = 0 disables the temporal term */
    float dropout_p;         /* 0 in eval mode */
    uint64_t seed;           /* dropout stream ; the mask is a pure function of (seed, layer_index, site, element) */
    const uint64_t* seed_dev;/* nullable DEVICE counter added to seed at kernel start: bump it per step so that a captured
                                CUDA graph draws a fresh mask on every replay */
    int layer_index;
} grb_hstu_dims;

typedef struct {
    const void* proj_w;      /* bf16 [4D, D]   layers.i.projection.weight (order U,V,Q,K along rows) */
    const float* proj_b;     /* [4D] */
    const float* pos_table;  /* [npos, H]      layers.i.position_bias.relative_attention_bias.weight */
    const float* time_table; /* [ntime, H] or NULL   layers.i.temporal_bias.temporal_attention_bias.weight */
    const float* ln1_g;      /* attn_norm */
    const float* ln1_b;
    const void* ffn1_w;      /* bf16 [4D, D]   ffn.0.weight */
    const float* ffn1_b;
    const void* ffn2_w;      /* bf16 [D, 4D]   ffn.3.weight */
    const float* ffn2_b;
    const float* ln2_g;      /* ffn_norm */
    const float* ln2_b;
} grb_hstu_layer_params;

typedef struct {             /* fp32, same shapes as the parameters, accumulated */
    float* proj_w; float* proj_b; float* pos_table; float* time_table;
    float* ln1_g; float* ln1_b; float* ffn1_w; float* ffn1_b; float* ffn2_w; float* ffn2_b; float* ln2_g; float* ln2_b;
} grb_hstu_layer_grads;

typedef struct {
    const uint16_t* bias_index; /* LEGACY (mma.sync) attention path only, NULL otherwise: [B, L, ld_index] from grb_hstu_bias_index():
                                   pos_bucket(i-j)*64 + time_bucket(|ts_i-ts_j|), or npos*64 for a masked cell (j > i, padded key) */
    int ld_index;               /* row pitch in ELEMENTS: a multiple of 8, >= L */
    int has_time;               /* 0: timestamps were None -> the temporal term is dropped (hstu.py:251) */
    int pos_uniform;            /* 1 when every delta in [0, L) maps to the same position bucket (the reference's behaviour):
                                   a bias_index, if given, must then have been built with npos = 1 and an all-zero pos_bucket table */
    int pos_bucket0;            /* that bucket (row of the [npos, H] table that is live) */
    /* per-sequence metadata: pad flags and timestamps (with their int32 rebasing for the bucket test hook) */
    const int64_t* timestamps;  /* [B, L] or NULL */
    const uint8_t* pad;         /* [B, L], 1 = input_ids == 0 */
    const int32_t* rel32;       /* [B, L] from grb_hstu_seq_prepare() (NULL when timestamps is NULL) */
    const uint8_t* wide;        /* [B]    from grb_hstu_seq_prepare() */
    const int64_t* time_thr;    /* [65] integer thresholds of the reference's fp32 log/0.693 bucket expression (see below) */
} grb_hstu_seq;

/* Per-sequence rebasing of the int64 timestamps (replaces nothing in the reference: it makes `ts[b,i] - ts[b,j]`
 * (hstu.py:400) a 32-bit subtraction in the in-kernel bucket routine): rel32[b,i] = ts[b,i] - min over non-padded positions;
 * wide[b] = 1 when the sequence spans >= 2^31 ticks, in which case the kernels use the int64 values themselves. */
int grb_hstu_seq_prepare(const int64_t* timestamps, const uint8_t* pad, int B, int L, int32_t* rel32, uint8_t* wide, void* stream);
/* Test hook: the time bucket / mask byte of every cell, [B, L, L] uint8 (bucket, or 64 when j > i or key j is padded), computed
 * by the in-kernel bucket routine from the rebased timestamps. */
int grb_hstu_bucket_bytes_debug(const grb_hstu_seq* s, int B, int L, int ntime, uint8_t* out, void* stream);
/* The attention core alone (hstu.py:244-267) on the projection output P = [U | V | Q | K] ([T, 4D] bf16): O [T, D] bf16.
 * backward: dO [T, D] bf16, zp [T, 4D] the pre-activations of P -> dzp columns V, Q, K (gradients w.r.t. the pre-activations),
 * bias-table gradients accumulated.  scratch: grb_hstu_attention_scratch_bytes(). */
size_t grb_hstu_attention_scratch_bytes(const grb_hstu_dims* d);
int grb_hstu_attention_forward(const grb_hstu_dims* d, const float* pos_table, const float* time_table, const grb_hstu_seq* s,
                               const void* P_bf16, void* O_bf16, void* stream);
int grb_hstu_attention_backward(const grb_hstu_dims* d, const float* pos_table, const float* time_table, const grb_hstu_seq* s,
                                const void* P_bf16, const void* zp_bf16, const void* dO_bf16, void* dzp_bf16, float* dpos_table,
                                float* dtime_table, void* scratch, void* stream);

/* Per-batch integer preprocessing shared by all layers / heads / passes (replaces the index arithmetic of
 * RelativePositionBias._relative_position_bucket (hstu.py:300-328), TemporalBias._temporal_bucket (:368-384) and the two
 * masked_fill's (:256-259)):
 *   tb        = clamp(trunc(log_f32(max(1,|ts_i - ts_j|)) / 0.693), 0, ntime-1)    (0 when timestamps == NULL)
 *   out[b,i,j] = (j <= i && !pad[b,j]) ? pos_bucket[i-j] * 64 + tb : npos * 64
 * tb is evaluated exactly through integer thresholds: time_thr[k] = smallest |dt| whose reference bucket is >= k (k < 64),
 * time_thr[64] = INT64_MAX.  pos_bucket: [L] bucket of delta = i - j >= 0, precomputed by the host from the reference
 * formula.  pad: [B, L], 1 = input_ids == 0. */
int grb_hstu_bias_index(const int64_t* timestamps, const uint8_t* pad, const int64_t* time_thr, const uint8_t* pos_bucket, int B,
                        int L, int npos, int ntime, uint16_t* out, int ld_index, void* stream);

/* Weight-gradient GEMMs (dW of a block, dE of the head) off the critical path: with grb_set_defer_weight_grads(1) they are enqueued
 * on a library-owned side stream, forked from the caller's stream where their operands are ready, and become visible to the
 * caller's stream only after grb_join_deferred(stream).  The caller must keep the operand buffers of the deferred work (the
 * `workspace` and `saved` blobs of grb_hstu_layer_backward, the workspace of grb_head_loss_forward_backward) alive until then.
 * CUDA-graph capturable (event fork / join).  Off by default: every entry point is then complete when its stream work is. */
int grb_set_defer_weight_grads(int on);
int grb_join_deferred(void* stream);

size_t grb_hstu_layer_saved_bytes(const grb_hstu_dims* d);
size_t grb_hstu_layer_workspace_bytes(const grb_hstu_dims* d);
int grb_hstu_layer_forward(const grb_hstu_dims* d, const grb_hstu_layer_params* p, const grb_hstu_seq* s,
                           const float* x, float* y, void* saved, void* stream);
int grb_hstu_layer_backward(const grb_hstu_dims* d, const grb_hstu_layer_params* p, const grb_hstu_seq* s,
                            const float* dy, const void* saved, float* dx, const grb_hstu_layer_grads* g,
                            void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------------ cached incremental inference
 * Extends `predict` / evaluation (hstu.py:150-157, trainers/hstu_trainer.py:55-81), which rerun the whole history for every new
 * item: a cache keeps, per layer, the K | V rows of every item seen so far for a batch of B users, and a chunk of n new slots per
 * user runs through the blocks against it.  Causal attention and relative-only biases make a cached row exact: for a left-padded
 * history the result equals the full forward's.  Inference only (no dropout, no backward).
 * Positions count items, not slots: the pads of a chunk are compacted away. */
typedef struct {
    int B, capacity, num_layers; /* capacity <= 16384 items per user */
    void* kv;                    /* bf16 [num_layers, B, capacity, 2D]: row p of user b = K | V of the user's p-th item */
    int64_t* timestamps;         /* [B, capacity] */
    int32_t* lengths;            /* [B] items cached per user */
    uint8_t* overflow;           /* [B] set to 1 when an item did not fit in `capacity` (it is dropped, never written) */
} grb_hstu_cache;
/* One launch per chunk, before the layers: input_ids / timestamps [B, n] (timestamps may be NULL -> 0 is stored; ids == 0 are
 * pads).  positions [B, n] int32 = the cache position of every valid row (-1 for a pad or a dropped item); the chunk's timestamps
 * are stored, lengths advance (never past capacity) and last_row [B] int32 = the chunk row of each user's last valid item, or -1. */
int grb_hstu_cache_append(const grb_hstu_cache* c, const int64_t* input_ids, const int64_t* timestamps, int n, int32_t* positions,
                          int32_t* last_row, void* stream);
/* One block on the chunk: d->L = n (dropout_p must be 0), x / y [B * n, D] fp32.  The K | V of the chunk's valid rows are written
 * into layer `layer` of the cache, then every valid row attends to the cached keys [0, position] of its user.
 * pos_bucket [capacity] uint8: position bucket of delta = p_i - p_j (the table RelativePositionBias.bucket_of_delta builds), or
 * NULL when every delta maps to bucket pos_bucket0 (the reference's behaviour).  time_thr [65] as in grb_hstu_bias_index; the
 * temporal term is used when d->ntime > 0 and p->time_table != NULL.  workspace: grb_hstu_layer_extend_workspace_bytes(d, capacity). */
size_t grb_hstu_layer_extend_workspace_bytes(const grb_hstu_dims* d, int capacity);
int grb_hstu_layer_extend(const grb_hstu_dims* d, const grb_hstu_layer_params* p, const grb_hstu_cache* c, int layer,
                          const int32_t* positions, const uint8_t* pos_bucket, int pos_bucket0, const int64_t* time_thr,
                          const float* x, float* y, void* workspace, void* stream);

/* Paged pool: the K | V rows of many users share one pool of pages, each user has a page table, and any set of distinct users
 * can be extended in one call, so memory follows the items actually cached rather than a per-user capacity.  Item p of user u
 * lives in page page_table[u, p / page_size] at row p % page_size.  The dense grb_hstu_cache is the pool with
 * page_size = capacity whose page b belongs to user b; both run on the same kernels.
 * Initial state: lengths, overflow and errors 0, free_stack = any permutation of 0 .. num_pages-1 (the next page handed out is
 * free_stack[*free_top - 1]), *free_top = num_pages, row_of filled with INT32_MAX (the allocation kernels leave it so). */
typedef struct {
    int max_users, num_layers;
    int page_size;               /* items per page: a positive multiple of 64 */
    int num_pages;
    int max_items;               /* most items one user can hold, <= 16384 */
    void* kv;                    /* bf16 [num_layers, num_pages, page_size, 2D] */
    int64_t* timestamps;         /* [num_pages, page_size] */
    int32_t* page_table;         /* [max_users, ceil(max_items / page_size)] */
    int32_t* lengths;            /* [max_users] items cached per user */
    uint8_t* overflow;           /* [max_users] 1 when an item of the user was dropped (no room within max_items or no free page) */
    int32_t* free_stack;         /* [num_pages] */
    int32_t* free_top;           /* [1] number of free pages */
    uint32_t* errors;            /* [1] bit 0: a row named a user outside [0, max_users); bit 1: a row repeated an earlier row's user */
    int32_t* row_of;             /* [max_users] scratch of the allocation kernels */
} grb_hstu_pool;
/* One call per chunk, before the layers: users [B] int64, input_ids / timestamps [B, n] as in grb_hstu_cache_append.  One CTA
 * validates the users (a row whose user is out of range or repeats an earlier row's is treated as all padding and sets a bit
 * of *errors), then hands out the pages the rows' new items need from the free stack, in row order; items beyond max_items or
 * without a page are dropped and flag their user in overflow.  Outputs as grb_hstu_cache_append, plus room [B] int32: the items
 * the row's user may hold after the allocation, -1 for a rejected row. */
int grb_hstu_pool_append(const grb_hstu_pool* pool, const int64_t* users, int B, const int64_t* input_ids, const int64_t* timestamps,
                         int n, int32_t* positions, int32_t* last_row, int32_t* room, void* stream);
/* Forgets users [B]: their pages go back onto the free stack (row order, then page order), their length and overflow flag become
 * 0, and so do their rows of last_hidden [max_users, D] fp32 (nullable; a caller-side buffer of per-user state).  Rows are
 * validated as in grb_hstu_pool_append. */
int grb_hstu_pool_release(const grb_hstu_pool* pool, const int64_t* users, int B, float* last_hidden, int D, void* stream);
/* grb_hstu_layer_extend on a pool: d->B = the call's rows, users [B] and positions [B, n] as given to / returned by
 * grb_hstu_pool_append; pos_bucket [max_items] or NULL.  The key split is a function of d and max_items only, so a captured graph
 * stays valid while lengths and page tables change on the device. */
size_t grb_hstu_layer_extend_paged_workspace_bytes(const grb_hstu_dims* d, const grb_hstu_pool* pool);
int grb_hstu_layer_extend_paged(const grb_hstu_dims* d, const grb_hstu_layer_params* p, const grb_hstu_pool* pool, int layer,
                                const int64_t* users, const int32_t* positions, const uint8_t* pos_bucket, int pos_bucket0,
                                const int64_t* time_thr, const float* x, float* y, void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------------ input pipeline
 * Device-side hstu_collate_fn / sasrec_collate_fn (genrec/data/amazon_hstu.py:137-173, genrec/data/amazon_sasrec.py:125-161): a
 * jagged batch (items / stamps [N] in time order, offsets [B+1], one held-out target per user) -> the LEFT-padded [B, L]
 * input_ids / targets (inputs shifted by one) / timestamps the models consume.  L = min(longest history of the batch, max_seq_len)
 * is chosen by the caller, who knows the lengths when it forms the batch.  stamps / out_timestamps may be NULL. */
int grb_collate_jagged(const int64_t* items, const int64_t* stamps, const int64_t* offsets, const int64_t* targets, int B, int L,
                       int64_t* out_input_ids, int64_t* out_targets, int64_t* out_timestamps, void* stream);

/* ------------------------------------------------------------------------------------------------ embedding gather
 * Replaces item_embedding + emb_dropout (hstu.py:124-128) / the scaled item+position embedding of SASRec
 * (sasrec.py:100-111).  pos_table may be NULL; mask_pad_rows multiplies rows whose id is 0 by zero (SASRec). */
int grb_embed_forward(const int64_t* ids, const float* table, const float* pos_table, float* x, uint8_t* pad,
                      int B, int L, int D, float scale, int mask_pad_rows, float dropout_p, uint64_t seed, const uint64_t* seed_dev,
                      void* stream);
/* order: the B * L token indices sorted by id (stable); every table row is summed over its tokens in token order, in a fixed
 * schedule (scratch: [B * L, D] fp32) - the gradient is the same from run to run */
int grb_embed_backward(const int64_t* ids, const int64_t* order, const float* dx, float* dtable, float* dpos_table, int B, int L, int D,
                       float scale, int mask_pad_rows, float dropout_p, uint64_t seed, const uint64_t* seed_dev, float* scratch,
                       void* stream);

/* ------------------------------------------------------------------------------------------------ tied-embedding head
 * Replaces final_norm + `x @ item_embedding.weight.T` + cross_entropy(ignore_index=0) (hstu.py:134-146,
 * sasrec.py:118-128) and their backward.  C = num_items + 1 classes. */
size_t grb_head_workspace_bytes(int T, int D, int C);
/* training: loss (scalar, mean over targets != 0), dx [T,D], and the three parameter gradients (accumulated). */
int grb_head_loss_forward_backward(const float* x, const float* ln_g, const float* ln_b, float ln_eps,
                                   const void* table_bf16, const int64_t* targets, int T, int D, int C, float* loss,
                                   float* dx, float* dtable, float* dln_g, float* dln_b, void* workspace, void* stream);
/* inference / API parity: logits fp32 [T, C] (contiguous), optional loss. */
int grb_head_logits(const float* x, const float* ln_g, const float* ln_b, float ln_eps, const void* table_bf16, int T,
                    int D, int C, float* logits, void* workspace, void* stream);

/* Leave-one-out evaluation without host round trips (replaces the per-sample loop of genrec/trainers/hstu_trainer.py:55-81):
 * logits [B, C] fp32 of the LAST position, targets [B] (0 = skip).  The rank of the target among classes 1..C-1 (class 0 is
 * excluded as the trainer's `logits[:, 0] = -inf` does) is counted on the device and the metric sums are ACCUMULATED:
 * metrics[0..2] += Recall@{1,5,10} hits, metrics[3..5] += NDCG@{1,5,10}.  ranks [B] int32 is optional. */
int grb_eval_rank_metrics(const float* logits, const int64_t* targets, int B, int C, float* metrics, int32_t* ranks, void* stream);

/* ------------------------------------------------------------------------------------------------ SASRec attention
 * Replaces MultiHeadAttention.forward (genrec/models/sasrec.py:192-246) after the three projections:
 *   out = softmax_j(mask(Q K^T * dh^-1/2)) * query_mask @ V     (residual and projections are GEMM epilogues) */
typedef struct {
    int B, L, D, H;
    float dropout_p; uint64_t seed; const uint64_t* seed_dev; int layer_index;
} grb_sasrec_dims;
int grb_sasrec_attention_forward(const grb_sasrec_dims* d, const void* q, const void* k, const void* v,
                                 const uint8_t* pad, void* out, float* lse, void* stream);
int grb_sasrec_attention_backward(const grb_sasrec_dims* d, const void* q, const void* k, const void* v,
                                  const uint8_t* pad, const void* out, const float* lse, const void* dout, void* dq,
                                  void* dk, void* dv, void* stream);

/* ------------------------------------------------------------------------------------------------ generic fused linear pieces
 * (used by the SASRec block and by tests)   act: 0 none, 1 silu, 2 relu */
int grb_linear_forward(const void* x_bf16, const void* w_bf16, const float* bias, int T, int N, int K, int act,
                       void* z_bf16, void* act_bf16, float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t site,
                       void* stream);
int grb_linear_residual_forward(const void* x_bf16, const void* w_bf16, const float* bias, const float* residual,
                                const float* row_scale, int T, int N, int K, float* y, float dropout_p, uint64_t seed,
                                const uint64_t* seed_dev, uint32_t site, void* stream);
/* dx[T,K] (+res) = dy[T,N] @ W[N,K] ; dW[N,K] += dy^T x ; db[N] += colsum(dy).  dW and db are summed in a fixed order, so they
 * are the same from run to run.  workspace: grb_linear_backward_workspace_bytes(T, N, K) bytes, required when dw or db is non-NULL. */
size_t grb_linear_backward_workspace_bytes(int T, int N, int K);
int grb_linear_backward(const void* dy_bf16, const void* w_bf16, const void* x_bf16, int T, int N, int K,
                        float* dx_f32, const float* dx_residual, float* dw, float* db, void* workspace, void* stream);
/* g[T,K] bf16 = dropmask(dy[T,N] @ W[N,K]) * act'(z[T,K])   (backward through `act(dropout)` of a hidden layer) ; act 1 silu, 2 relu */
int grb_linear_dact_backward(const void* dy_bf16, const void* w_bf16, const void* z_bf16, int T, int N, int K, int act,
                             float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t site, void* g_bf16, void* stream);
/* out_bf16[t,:] = bf16(dropmask(in[t,:]) * row_scale[t])   (row_scale may be NULL) */
int grb_cast_rows_f32_to_bf16(const float* in, void* out_bf16, int T, int D, const float* row_scale, float dropout_p, uint64_t seed,
                              const uint64_t* seed_dev, uint32_t site, void* stream);
int grb_layernorm_forward(const float* x, const float* g, const float* b, float eps, int T, int D, void* y_bf16,
                          float* y_f32, float* stats, void* stream);
/* dx = LayerNorm backward of dy (+ residual) ; dg, db += in a fixed order.  workspace: grb_layernorm_backward_workspace_bytes(T, D). */
size_t grb_layernorm_backward_workspace_bytes(int T, int D);
int grb_layernorm_backward(const float* dy, const float* x, const float* stats, const float* g, const float* residual,
                           int T, int D, float* dx, float* dg, float* db, void* workspace, void* stream);

/* fp32-accurate linear layer on the bf16 tensor path (the RQ-VAE encoder MLP, genrec/modules/encoder.py:399-420: bias-free
 * Linear + SiLU).  Operands are split into three bf16 terms each and the six significant cross terms are laid out along K
 * (K' = 6 K), so one wgmma GEMM with fp32 accumulation reproduces the fp32 product to ~2^-22 relative.
 *   grb_split3_f32_to_bf16: in [rows, K] fp32 -> out [rows, 6 K] bf16 ; operand 0 = activation (A) layout, 1 = weight (B) layout
 *   grb_linear_f32x3_forward: y [T, N] fp32 = act(x [T, K] @ W [N, K]^T), both operands pre-split ; act 0 none, 1 silu */
int grb_split3_f32_to_bf16(const float* in, void* out_bf16, size_t rows, int K, int operand, void* stream);
int grb_linear_f32x3_forward(const void* x_split_bf16, const void* w_split_bf16, int T, int N, int K, int act, float* y, void* stream);
/*   grb_linear_f32x3_bias_forward: y [T, ldy] fp32 = act(x @ W^T + bias) + residual ; bias [N] and residual [T, ldy] may be NULL,
 *   ldy >= N a multiple of 4 (the tied head has N = V + 1) */
int grb_linear_f32x3_bias_forward(const void* x_split_bf16, const void* w_split_bf16, const float* bias, const float* residual, int T,
                                  int N, int K, int act, float* y, int ldy, void* stream);

/* ------------------------------------------------------------------------------------------------ fp32-exact HSTU block (forward)
 * What the reference computes WITHOUT autocast (plain fp32 modules, hstu.py:222-280), for the "1e-5 (fp32)" parity target:
 * every linear layer is the split-bf16 GEMM above, attention / LayerNorm / gating are fp32 CUDA-core kernels
 * (csrc/exact_f32.cuh).  Forward only - evaluation, inference and parity; dropout is the identity.  The weight matrices arrive
 * pre-split (grb_split3_f32_to_bf16, operand 1): proj [4D, 6D], ffn1 [4D, 6D], ffn2 [D, 24D].  `s` must carry the
 * [B, L, ld_index] bias index matrix of grb_hstu_bias_index(). */
typedef struct {
    const void* proj_w_split; const float* proj_b;
    const float* pos_table; const float* time_table;   /* [npos, H], [ntime, H] or NULL */
    const float* ln1_g; const float* ln1_b;
    const void* ffn1_w_split; const float* ffn1_b;
    const void* ffn2_w_split; const float* ffn2_b;
    const float* ln2_g; const float* ln2_b;
} grb_hstu_layer_params_f32;
size_t grb_hstu_layer_f32_workspace_bytes(const grb_hstu_dims* d);
int grb_hstu_layer_forward_f32(const grb_hstu_dims* d, const grb_hstu_layer_params_f32* p, const grb_hstu_seq* s, const float* x, float* y,
                               void* workspace, void* stream);
/* y [T, D] fp32 = LayerNorm(x) in fp32 (the final norm in front of the fp32 head, hstu.py:134) */
int grb_layernorm_f32_forward(const float* x, const float* g, const float* b, float eps, int T, int D, float* y, void* stream);

/* ------------------------------------------------------------------------------------------------ T5-style attention core (TIGER)
 * The score / softmax / value part of T5Attention.forward (genrec/modules/transformer.py:133-156), between the q / k / v and the
 * output projections:  softmax((q k^T) scale + rel_bias[h, bucket(j - i)], key padding -> -1e9, causal -> -inf) with dropout on
 * the weights, times v.  q [B, Lq, ldq], k / v [B, Lk, ld] and out are bf16 with head h in columns h*head_dim .. ; bias [H,
 * num_buckets] fp32 with bucket [Lq + Lk - 1] int32 = the bucket of delta = j - i at index delta + Lq - 1 (both NULL for
 * cross-attention); key_pad [B, Lk] 1 = padded (NULL: none); lse [B, H, Lq, 2] = {row max, sum of exp(s - max)} is saved for the backward.
 * Backward: dq bf16 [B, Lq, lddq]; dk, dv fp32 [B, Lk, H * head_dim] (zero-filled here, then accumulated); dbias [H, num_buckets] +=. */
int grb_t5_attention_forward(const void* q, const void* k, const void* v, int B, int Lq, int Lk, int H, int head_dim, int ldq, int ldk, int ldv,
                             const float* bias, const int32_t* bucket, int num_buckets, const uint8_t* key_pad, int causal, float scale,
                             float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t site, void* out, int ldo, float* lse,
                             void* stream);
int grb_t5_attention_backward(const void* q, const void* k, const void* v, int B, int Lq, int Lk, int H, int head_dim, int ldq, int ldk, int ldv,
                              const float* bias, const int32_t* bucket, int num_buckets, const uint8_t* key_pad, int causal, float scale,
                              float dropout_p, uint64_t seed, const uint64_t* seed_dev, uint32_t site, const void* out, int ldo,
                              const float* lse, const void* dout, int lddo, void* dq, int lddq, float* dk, float* dv, float* dbias,
                              void* stream);

/* ------------------------------------------------------------------------------------------------ TIGER constrained beam step
 * The per-step post-processing of Tiger.generate (genrec/models/tiger.py:364-441), host-bound Python loops in the reference.
 * Trie = CSR over node ids: child_off [n_nodes + 1], child_tok / child_node [n_edges] sorted by token inside a node; root = 0,
 * dead = -1 (genrec_b200.tiger_decode.TrieCSR builds it from valid_item_ids, the reference's build_trie, tiger.py:49-69).
 *   grb_trie_log_softmax: logits [rows, V] -> probs, logp [rows, V] = softmax / log_softmax(masked_fill(~legal, -1e32) / temperature);
 *       legal = vocab_offset + the children of node[row] (use_trie), or the range [vocab_offset, vocab_offset + num_embeddings) with
 *       -inf elsewhere (use_trie = 0, tiger.py:377-381).
 *   grb_beam_select: total = beam_logps + cand_logp, sorted descending (equal totals: lower flat index first); the first K candidates
 *       whose token sequence is new survive; missing ones become (zeros, -1e32, root).  cand_tok are raw token ids (vocabulary index
 *       - vocab_offset).  new_nodes / nodes NULL without a trie.  K <= 32, K * KK <= 1024. */
int grb_trie_log_softmax(const float* logits, int rows, int V, const int32_t* node, const int32_t* child_off, const int32_t* child_tok,
                         int n_nodes, int use_trie, int vocab_offset, int num_embeddings, float temperature, float* probs, float* logp,
                         void* stream);
int grb_beam_select(const int64_t* beam_seqs, const float* beam_logps, const int64_t* cand_tok, const float* cand_logp, const int32_t* nodes,
                    const int32_t* child_off, const int32_t* child_tok, const int32_t* child_node, int n_nodes, int B, int K, int KK, int S,
                    int64_t* new_seqs, float* new_logps, int32_t* new_nodes, void* stream);

/* ------------------------------------------------------------------------------------------------ optimizer / casts */
int grb_cast_f32_to_bf16(const float* in, void* out_bf16, size_t n, void* stream);
/* torch.optim.Adam semantics on a flat buffer; state = 3 floats {step, 1-b1^step, 1-b2^step} ticked ON DEVICE. */
int grb_adam_step(float* p, float* g, float* m, float* v, void* p_bf16, size_t n, float* state, float lr, float beta1,
                  float beta2, float eps, float weight_decay, float grad_scale, int zero_grad, void* stream);

/* Device-side contract check: traps (asynchronous CUDA error at the next synchronisation) unless *value == 1.0f.  Used by the
 * opt-in "unit loss gradient" fast path, where parameter gradients are accumulated into the flat buffer before the incoming
 * gradient of the loss is known. */
int grb_assert_unit_scalar(const float* value, void* stream);

/* Data-parallel optimizer step over NVLink peer memory, replacing `all_reduce(grad)` + Adam (the DDP gradient all-reduce of
 * accelerator.backward, genrec/trainers/hstu_trainer.py:159, + optimizer.step, :160): cross-GPU barrier, then each rank reduces ITS
 * slice of the flat gradient over all ranks (multimem.ld_reduce through the NVSwitch when mc_* are given, peer loads otherwise),
 * applies Adam to the slice and stores the new fp32 parameters and their bf16 mirror to every rank (multimem.st / peer stores),
 * barrier, gradient zeroed.  All buffers are symmetric allocations of n elements, n % (8 * world) == 0.
 *   peer_g / peer_p / peer_mirror / peer_sig: DEVICE arrays of `world` pointers (rank order) ; mc_*: multicast addresses or NULL
 *   sig: this rank's flag words [2][world] (zero-initialised symmetric memory) ; epoch: 2 local counters (zero-initialised)
 *   state: as grb_adam_step (ticked here).  grad_scale = 1/world reproduces DDP's gradient averaging. */
int grb_dp_adam_step(float* p, float* g, float* m, float* v, void* p_bf16, const void* mc_g, void* mc_p, void* mc_p_bf16,
                     const void* peer_g, const void* peer_p, const void* peer_p_bf16, const void* peer_sig, void* sig, void* epoch,
                     size_t n, int rank, int world, float* state, float lr, float beta1, float beta2, float eps, float weight_decay,
                     float grad_scale, void* stream);

/* ------------------------------------------------------------------------------------------------ RQ-VAE residual argmin
 * Replaces the Quantize.forward distance+argmin (genrec/models/rqvae.py:185-199, eval branch :246-248) iterated by
 * RqVae.get_semantic_ids (:397-412).  x [N, D] fp32 latent, codebooks [levels, K, D] fp32.
 * ids [N, levels] int64 ; optional emb / res [N, D, levels] (reference layout), loss [N], res_out [N, D]. */
int grb_rq_residual_argmin(const float* x, const float* codebooks, int64_t N, int D, int K, int levels,
                           float commitment, int64_t* ids, float* emb, float* res, float* loss, float* res_out,
                           void* stream);

/* ------------------------------------------------------------------------------------------------ RQ-VAE training
 * Sinkhorn-Knopp hard assignment of the SINKHORN estimator (genrec/models/rqvae.py:85-110, :218-241) in one launch of one
 * thread-block cluster.  dist [B, K] fp32 distances of the level; 1 <= B, 2 <= K <= 256 (B = 0 returns 0).  In fp32:
 * mid = (max + min) / 2, amp = (max - mid) + 1e-5, dn = (dist - mid) / amp; then fp64: K = exp(-dn / eps), v = 1,
 * `iters` x { u = r / (K v + 1e-8); v = c / (K^T u + 1e-8) } with r = (float)(1/B), c = (float)(1/K);
 * ids[i] = argmax_j (u_i K_ij) v_j (first index on ties).  u_out [B] / v_out [K] (nullable) receive the final u and v.
 * Deterministic (fixed-order sums), graph-capturable; the workspace holds u and, when a CTA's rows of K do not fit shared memory,
 * K itself.  GRB_ENODEV when one cluster of 16 CTAs does not fit the device. */
size_t grb_rq_sinkhorn_workspace_bytes(int64_t B, int K);
int grb_rq_sinkhorn(const float* dist, int64_t B, int K, double eps, int iters, int64_t* ids, double* u_out, double* v_out,
                    void* workspace, void* stream);

/* One Lloyd step of the k-means codebook initialisation (genrec/modules/kmeans.py:58-76) after the assignment: for every cluster c
 * of the k, counts[c] = rows with assign == c; a non-empty cluster's centroid [c, :] becomes the mean of its rows (fixed-order fp64
 * sum, rounded to fp32) and shift[c] = |new - old|; an empty one is left as it was (shift[c] = 0) for the caller to reseed.
 * x [B, D] fp32, 1 <= D <= 256, assign [B] int64 in [0, k), centroids [k, D] fp32 updated in place. */
int grb_kmeans_update(const float* x, const int64_t* assign, int64_t B, int D, int k, float* centroids, int32_t* counts, float* shift,
                      void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GENREC_B200_H */
