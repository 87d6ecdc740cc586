/*
 * tzk.h — C-ABI of the H100-native sparse-embedding + feature-interaction engine.
 *
 * This is the drop-in boundary (SURVEY.md §8b).  Every entry point replaces one operator that the
 * reference reaches through third-party wheels (torchrec 1.7.0 / fbgemm-gpu 1.7.0, pinned in
 * requirements/runtime.txt:5,25 of the reference) or plain ATen; the call site inside the reference is
 * cited on each declaration (paths relative to the reference checkout (alibaba/TorchEasyRec @ 54cac316)).
 *
 * Conventions
 *  - extern "C", plain pointers and sizes, no torch types.  All pointers are DEVICE pointers unless the
 *    parameter name ends in `_host`.
 *  - The library never allocates or frees device memory: callers pass outputs and a workspace
 *    (`tzk_*_workspace_bytes` tells how big).
 *  - Every call only enqueues work on `stream` (a cudaStream_t passed as void*) and returns; no host sync,
 *    so every call is CUDA-graph capturable.
 *  - Return 0 on success, non-zero on failure; `tzk_last_error()` returns a thread-local message.
 *  - fp32 tables / fp32 accumulate; ids int64; lengths int32; offsets int64 (KJT layout of
 *    tzrec/datasets/utils.py:299-342: values key-major, lengths[f*B + b]).
 *
 * "Feature descriptor" arrays (one entry per KJT key f, device memory, built once at module init):
 *    feat_w_off[f]   int64  element offset of the feature's table inside the shard arena `weights`
 *    feat_rows[f]    int64  number of rows of that (local shard of the) table
 *    feat_dim[f]     int32  embedding dim D_f (multiple of 4 is the fast path; any D >= 1 works)
 *    feat_col[f]     int32  first output column of the feature in the pooled row
 *    feat_pool[f]    int32  0 = SUM, 1 = MEAN
 *    feat_key_base[f] int64 first sort key of the feature's table (row r of the table has key base + r);
 *                           tables sharing a physical table share the base.
 */
#ifndef TZK_H_
#define TZK_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TZK_ABI_VERSION 1

#define TZK_POOL_SUM 0
#define TZK_POOL_MEAN 1

#define TZK_OPT_SGD 0             /* w -= lr*g                                   (App. A.10) */
#define TZK_OPT_ADAGRAD 1         /* s += g*g ; w -= lr*g/(sqrt(s)+eps)          (EXACT_ADAGRAD) */
#define TZK_OPT_ROWWISE_ADAGRAD 2 /* s_row += mean_d(g*g) ; w -= lr*g/(sqrt(s_row)+eps) */
/* the next two only through tzk_fused_bwd_ex / tzk_fused_bwd_apply_ex (they need tzk_opt_args) */
#define TZK_OPT_ADAM 3            /* m=b1 m+(1-b1)g ; v=b2 v+(1-b2)g*g ; w -= lr*(m^/(sqrt(v^)+eps) + wd*w)  (ADAM) */
#define TZK_OPT_PARTIAL_ROWWISE_ADAM 4 /* m element-wise, v one value per row from mean_d(g*g)  (PARTIAL_ROWWISE_ADAM) */
/* the layer-wise adaptive optimizers, also _ex only; |.| = L2 norm over the row's D elements */
#define TZK_OPT_LAMB 5            /* m, v as ADAM ; u = m^/(sqrt(v^)+eps) + wd*w ; w -= lr*(|w|/|u|)*u            (LAMB) */
#define TZK_OPT_PARTIAL_ROWWISE_LAMB 6 /* m element-wise, v one value per row from mean_d(g*g), u and step as LAMB (PARTIAL_ROWWISE_LAMB) */
#define TZK_OPT_LARS_SGD 7        /* lr' = lr*eta*|w|/(|g|+wd*|w|) ; m = momentum*m + lr'*(g+wd*w) ; w -= m   (LARS_SGD) */
/* peer-memory step only (_ex entry points): no update — weights[row] = summed gradient of the row, ((int32*)state)[key]
 * = 1; `weights` is then a dense per-row partial-sum buffer, not a table (see tzk_peer_small_update) */
#define TZK_OPT_ACCUM_OUT 100

/* Optimizer description for the _ex entry points (what tzrec/optim/optimizer_builder.py:30-97 passes to
 * apply_optimizer_in_backward; field names follow tzrec/protos/optimizer.proto:76-139).  Host struct, device
 * pointers inside.
 *   state  : SGD unused; ADAGRAD / ADAM / PARTIAL_ROWWISE_ADAM / LAMB / PARTIAL_ROWWISE_LAMB / LARS_SGD: same layout as
 *            `weights` (accumulator / first moment / momentum); ROWWISE_ADAGRAD: one float per key.
 *   state2 : ADAM / LAMB: second moment, same layout as `weights`; PARTIAL_ROWWISE_ADAM / PARTIAL_ROWWISE_LAMB: one float
 *            per key.  `step` as well: the LAMB variants use the same bias correction as Adam.
 *   step   : device scalar holding the 1-based iteration count of this update as a float (bias correction
 *            1 - beta^t is evaluated on the device, so a captured CUDA graph can keep replaying).
 *   max_gradient > 0 clamps every element of the summed row gradient to [-max_gradient, max_gradient]
 *   (gradient_clipping = true); weight_decay is fbgemm's: w -= lr * weight_decay * w inside the same update. */
typedef struct tzk_opt_args {
  int32_t optimizer;
  float lr, eps, beta1, beta2, weight_decay, max_gradient;
  float* state;
  float* state2;
  const float* step;
  int32_t weights_f16; /* 1: `weights` points to an arena of IEEE halfs (EmbeddingBagConfig.data_type = FP16,
                        * tzrec/protos/feature.proto data_type): rows are widened to fp32, updated, rounded to nearest */
  int32_t interleaved; /* 1 (fp32 tables, TZK_OPT_ADAGRAD): `weights` holds [weight row | accumulator row] back to back, row
                        * stride 2 * D_f elements (feat_w_off in those units): a D = 16 row and its state share one 128-B
                        * line, so the update reads and writes whole lines (two half-line writes cost a read-modify-write
                        * each in DRAM: profiles/README.md).  `state` is ignored.  Lookups over such an arena:
                        * tzk_pooled_gather_fwd_strided / tzk_seq_gather_fwd_strided. */
  float momentum, eta;  /* LARS_SGD: momentum of the velocity and the trust coefficient (fbgemm's default eta = 0.001) */
  int32_t weight_decay_mode; /* ROWWISE_ADAGRAD (tzrec WeightDecayMode): 0 NONE (weight_decay ignored); 1 L2:
                        * s_row += mean_d((g + wd*w)^2), w = (1 - mult*wd)*w - mult*g; 2 DECOUPLE: s_row += mean_d(g*g),
                        * w = (1 - lr*wd)*w - mult*g; mult = lr/(sqrt(s_row)+eps) */
  const float* per_sample_weights; /* NULL: unweighted bags.  Else weighted bags (pooled layout, [EXT] the weighted TBE
                        * backward, split_embedding_backward_codegen_*_weighted_exact): position l contributes
                        * grad_scale * w[l] * grad_out row (/ L for MEAN).  tzk_fused_bwd_ex reads w[nnz] here and needs
                        * tzk_fused_bwd_weighted_workspace_bytes; tzk_fused_bwd_apply_ex only checks it is non-NULL and
                        * consumes the workspace of tzk_fused_bwd_sort_weighted.  The peer entry points reject it. */
} tzk_opt_args;

typedef void* tzk_stream_t; /* cudaStream_t */

/* ---- misc --------------------------------------------------------------------------------------- */
int tzk_abi_version(void);
const char* tzk_last_error(void);
/* number of SMs of the current device (used by callers to size persistent grids); <0 on error */
int tzk_sm_count(void);

/* ---- K3: lengths -> offsets  ([EXT] fbgemm::asynchronous_complete_cumsum, implicit in every
 * KeyedJaggedTensor.offsets(); reached from tzrec/modules/embedding.py:930) -------------------------
 * offsets[0] = 0, offsets[i+1] = sum(lengths[0..i]).  n may be 0. */
size_t tzk_lengths_to_offsets_workspace_bytes(int64_t n);
int tzk_lengths_to_offsets(const int32_t* lengths, int64_t n, int64_t* offsets, void* workspace,
                           size_t workspace_bytes, tzk_stream_t stream);

/* ---- K4: pooled gather forward  ([EXT] fbgemm TBE split_embedding_codegen_forward_unweighted; the
 * reference call is `self.ebc(sparse_feature)` tzrec/modules/embedding.py:930) ------------------------
 * out[b, feat_col[f] : +D_f] = pool_{l in bag(f,b)} weights[feat_w_off[f] + ids[l]*D_f : +D_f]
 * bag(f,b) = [offsets[f*B+b], offsets[f*B+b+1]).  MEAN of an empty bag is 0.  Sequential fp32 add in
 * list order.  Ids outside [0, feat_rows[f]) read row 0 (fbgemm bounds_check WARNING mode, App. A.9).
 * Launch hints (host scalars, known at module init): max_dim = max_f D_f; vec_ok != 0 promises that every
 * D_f, feat_col[f] and feat_w_off[f] is a multiple of 4 (16-B vector path). */
int tzk_pooled_gather_fwd(const float* weights, const int64_t* feat_w_off, const int64_t* feat_rows,
                          const int32_t* feat_dim, const int32_t* feat_col, const int32_t* feat_pool,
                          const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B,
                          int32_t max_dim, int32_t vec_ok, float* out, int64_t ld_out,
                          tzk_stream_t stream);

/* ---- K4-nobag: un-pooled (sequence) gather  ([EXT] TBE ..._nobag; `ec(kjt)` embedding.py:1301) ------
 * out[l, 0:D] = weights[feat_w_off[f(l)] + ids[l]*D : +D]  for l in [0, nnz); every feature must have
 * the same dim D (the reference builds one EmbeddingCollection per dim, embedding.py:1193-1197).
 * f(l) is found from `offsets` (key boundaries offsets[f*B]). */
int tzk_seq_gather_fwd(const float* weights, const int64_t* feat_w_off, const int64_t* feat_rows,
                       const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B, int32_t D,
                       int64_t nnz, float* out, tzk_stream_t stream);

/* ---- strided tables: rows of feature f's table are feat_stride[f] >= D_f elements apart (NULL: dense rows) — the
 * interleaved [weight row | optimizer-state row] arena of tzk_opt_args.interleaved.  vec_ok additionally promises
 * that every stride is a multiple of 4.  Same reference call sites as K4 / K4-nobag above. */
int tzk_pooled_gather_fwd_strided(const float* weights, const int64_t* feat_w_off, const int64_t* feat_rows,
                                  const int32_t* feat_dim, const int32_t* feat_stride, const int32_t* feat_col,
                                  const int32_t* feat_pool, const int64_t* ids, const int64_t* offsets, int32_t F,
                                  int32_t B, int32_t max_dim, int32_t vec_ok, float* out, int64_t ld_out,
                                  tzk_stream_t stream);
int tzk_seq_gather_fwd_strided(const float* weights, const int64_t* feat_w_off, const int64_t* feat_rows,
                               const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B, int32_t D,
                               int32_t row_stride, int64_t nnz, float* out, tzk_stream_t stream);

/* ---- FP16 tables (tzrec/protos/feature.proto `data_type = "FP16"` -> EmbeddingBagConfig.data_type, features/feature.py:
 * 626,652): the same lookups over an arena of IEEE halfs; pooling and outputs stay fp32.  The fused backward takes such
 * an arena through tzk_opt_args.weights_f16 (the _ex entry points); optimizer state stays fp32.  Sharded collections
 * keep their shards as halfs too: the peer step's _f16 entry points at the end of this header. */
int tzk_pooled_gather_fwd_f16(const void* weights, const int64_t* feat_w_off, const int64_t* feat_rows,
                              const int32_t* feat_dim, const int32_t* feat_col, const int32_t* feat_pool,
                              const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B, int32_t max_dim,
                              int32_t vec_ok, float* out, int64_t ld_out, tzk_stream_t stream);
int tzk_seq_gather_fwd_f16(const void* weights, const int64_t* feat_w_off, const int64_t* feat_rows, const int64_t* ids,
                           const int64_t* offsets, int32_t F, int32_t B, int32_t D, int64_t nnz, float* out,
                           tzk_stream_t stream);

/* ---- K4w: weighted pooled gather  ([EXT] fbgemm TBE split_embedding_codegen_forward_weighted; torchrec's sharded
 * lookup passes `features.weights_or_none()` as per_sample_weights — IdFeature `weighted: true`,
 * tzrec/features/id_feature.py, tzrec/datasets/utils.py:299-342) ------------------------------------------------------
 * out[b, feat_col[f] : +D_f] = pool_{l in bag(f,b)} per_sample_weights[l] * row(ids[l]), accumulated in fp32 in list order
 * as acc = fmaf(w[l], row, acc) (the first term w[l0] * row), MEAN multiplies by 1/L at the end; with all-ones weights the
 * bits equal the unweighted lookup's.  One entry point for the three arena formats: weights_f16 != 0 -> halfs (like
 * tzk_pooled_gather_fwd_f16), else fp32 with dense rows (feat_stride NULL) or strided rows (like _strided). */
int tzk_pooled_gather_fwd_weighted(const void* weights, int32_t weights_f16, const int64_t* feat_w_off,
                                   const int64_t* feat_rows, const int32_t* feat_dim, const int32_t* feat_stride,
                                   const int32_t* feat_col, const int32_t* feat_pool, const int64_t* ids,
                                   const int64_t* offsets, const float* per_sample_weights, int32_t F, int32_t B,
                                   int32_t max_dim, int32_t vec_ok, float* out, int64_t ld_out, tzk_stream_t stream);

/* ---- K5: fused backward + sparse optimizer  ([EXT] TBE split_embedding_backward_codegen_*_exact,
 * installed by apply_optimizer_in_backward at tzrec/main.py:774-781; optimizer choice
 * tzrec/optim/optimizer_builder.py:30-97) -------------------------------------------------------------
 * For every table row touched by the batch: g = sum over all (bag, slot) hitting the row of
 * grad_scale * grad_out[b, feat_col[f] : +D] (MEAN bags contribute /L), then ONE optimizer update in
 * place.  Deterministic: contributions are ordered by a stable sort on (table,row).
 * `state`: ADAGRAD -> same layout as `weights`; ROWWISE_ADAGRAD -> one float per key (state[key]);
 * SGD -> ignored (may be NULL).
 * pooled == 0 selects the un-pooled (sequence) layout: grad_out is [nnz, D] indexed by id position.
 * A feature with feat_rows[f] == 0 is wire padding: its ids are sorted behind every real key and ignored.
 * total_keys = one past the largest sort key (sum of physical rows).  Requires nnz < 2^31. */
size_t tzk_fused_bwd_workspace_bytes(int64_t nnz, int64_t total_keys, int32_t max_dim);
int tzk_fused_bwd(int32_t optimizer, int32_t pooled, const float* grad_out, int64_t ld_grad,
                  const int64_t* feat_w_off, const int64_t* feat_rows, const int32_t* feat_dim,
                  const int32_t* feat_col, const int32_t* feat_pool, const int64_t* feat_key_base,
                  const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B, int64_t nnz,
                  int64_t total_keys, int32_t max_dim, int32_t vec_ok, float* weights, float* state,
                  float lr, float eps, float grad_scale, void* workspace, size_t workspace_bytes,
                  tzk_stream_t stream);
/* The same update in two calls that share `workspace` (tzk_fused_bwd_workspace_bytes): _sort needs only the ids, so
 * the host can enqueue it on a side stream as soon as the batch is on the device — it then overlaps the forward
 * pass (what TrainPipelineSparseDist does for the input dist, tzrec/utils/dist_util.py:221-303) — and _apply,
 * ordered after it, consumes the gradient.  tzk_fused_bwd == _sort followed by _apply on one stream. */
int tzk_fused_bwd_ex(const tzk_opt_args* opt, int32_t pooled, const float* grad_out, int64_t ld_grad,
                     const int64_t* feat_w_off, const int64_t* feat_rows, const int32_t* feat_dim,
                     const int32_t* feat_col, const int32_t* feat_pool, const int64_t* feat_key_base,
                     const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B, int64_t nnz,
                     int64_t total_keys, int32_t max_dim, int32_t vec_ok, float* weights, float grad_scale,
                     void* workspace, size_t workspace_bytes, tzk_stream_t stream);
int tzk_fused_bwd_apply_ex(const tzk_opt_args* opt, int32_t pooled, const float* grad_out, int64_t ld_grad,
                           const int64_t* feat_w_off, const int64_t* feat_rows, const int32_t* feat_dim,
                           const int32_t* feat_col, const int32_t* feat_pool, const int64_t* feat_key_base,
                           const int64_t* offsets, int32_t F, int32_t B, int64_t nnz, int64_t total_keys,
                           int32_t max_dim, int32_t vec_ok, float* weights, float grad_scale, void* workspace,
                           size_t workspace_bytes, tzk_stream_t stream);
int tzk_fused_bwd_sort(int32_t pooled, const int64_t* feat_rows, const int64_t* feat_key_base, const int64_t* ids,
                       const int64_t* offsets, int32_t F, int32_t B, int64_t nnz, int64_t total_keys,
                       int32_t max_dim, void* workspace, size_t workspace_bytes, tzk_stream_t stream);
int tzk_fused_bwd_apply(int32_t optimizer, int32_t pooled, const float* grad_out, int64_t ld_grad,
                        const int64_t* feat_w_off, const int64_t* feat_rows, const int32_t* feat_dim,
                        const int32_t* feat_col, const int32_t* feat_pool, const int64_t* feat_key_base,
                        const int64_t* offsets, int32_t F, int32_t B, int64_t nnz, int64_t total_keys,
                        int32_t max_dim, int32_t vec_ok, float* weights, float* state, float lr, float eps,
                        float grad_scale, void* workspace, size_t workspace_bytes, tzk_stream_t stream);

/* Weighted bags ([EXT] the weighted TBE backward, split_embedding_backward_codegen_*_weighted_exact, without the
 * gradient w.r.t. the weights): tzk_opt_args.per_sample_weights non-NULL, pooled layout only.  The workspace must have
 * tzk_fused_bwd_weighted_workspace_bytes.  tzk_fused_bwd_sort_weighted is the id half (it also leaves the weights in
 * sorted order in the workspace); tzk_fused_bwd_apply_ex with a non-NULL per_sample_weights is its gradient half. */
size_t tzk_fused_bwd_weighted_workspace_bytes(int64_t nnz, int64_t total_keys, int32_t max_dim);
int tzk_fused_bwd_sort_weighted(int32_t pooled, const int64_t* feat_rows, const int64_t* feat_key_base, const int64_t* ids,
                                const int64_t* offsets, const float* per_sample_weights, int32_t F, int32_t B,
                                int64_t nnz, int64_t total_keys, int32_t max_dim, void* workspace,
                                size_t workspace_bytes, tzk_stream_t stream);

/* ---- pooled-lookup backward w.r.t. a row buffer in which every row is referenced exactly once (the
 * sample owner's half of the sharded backward; our replacement of [EXT] PooledEmbeddingsAllToAll /
 * PooledEmbeddingsReduceScatter backward, App. A.6 / A.8):
 *   g_rows[slot[l], 0:D] = grad_out[b, feat_col[f] : +D] * (MEAN ? 1/L(f,b) : 1)   for every id position l
 * of bag (f,b).  All features share one dim D. */
int tzk_bag_grad_expand(const float* grad_out, int64_t ld_grad, const int32_t* feat_col,
                        const int32_t* feat_pool, const int64_t* offsets, const int32_t* slot, int32_t F,
                        int32_t B, int32_t D, float* g_rows, tzk_stream_t stream);

/* ---- K1: block bucketize  ([EXT] fbgemm::block_bucketize_sparse_features, reached through
 * DistributedModelParallel at tzrec/main.py:799; geometry App. A.5 / A.7) ----------------------------
 * dest r = feat_owner[f] + id / feat_block[f], local id = id - (id / feat_block[f]) * feat_block[f].
 *   row-wise   : owner 0, block = ceil(rows / W)
 *   table-wise : owner = rank holding the table, block >= rows (quotient 0, id unchanged)
 * feat_owner may be NULL (all 0).  Outputs, laid out [W][F][B] (dest-major):
 *   out_lengths[(r*F+f)*B + b]   number of ids of bag (f,b) that go to rank r
 *   out_offsets [W*F*B+1]         scan of out_lengths (by-product)
 *   out_ids                       local ids in that order; relative order inside a bag is kept
 *                                 (bucketize_pos = false)
 *   out_pos (nullable)            out_pos[o] = input position of output slot o ("unbucketize permute")
 *   out_inv (nullable)            out_inv[l] = output slot of input position l (its inverse)
 * wire_capacity = 0: compact layout as above.  wire_capacity = C > 0: fixed-capacity wire layout — the ids of
 * destination r occupy out_ids[r*C ...] (out_ids / out_pos then hold W*C slots, unused ones are left untouched,
 * so pre-fill them); ids that do not fit are dropped and the caller detects that from the counts. */
size_t tzk_bucketize_rw_workspace_bytes(int32_t F, int32_t B, int32_t W, int64_t nnz);
int tzk_bucketize_rw(const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B, int32_t W,
                     const int64_t* feat_block, const int32_t* feat_owner, int64_t nnz,
                     int64_t wire_capacity, int32_t* out_lengths, int64_t* out_offsets, int64_t* out_ids,
                     int32_t* out_pos, int32_t* out_inv, void* workspace, size_t workspace_bytes,
                     tzk_stream_t stream);

/* ---- K2: KJT segment permute  ([EXT] fbgemm::permute_2D_sparse_data, KeyedJaggedTensor.permute;
 * used by the TW input-dist, App. A.5) ----------------------------------------------------------------
 * Segment s (= key, or (rank,key)) of the output is segment perm[s] of the input; each segment has B
 * bags.  out_offsets [S_out*B+1] must already hold the scan of the permuted lengths (use
 * tzk_permute_lengths + tzk_lengths_to_offsets). */
int tzk_permute_lengths(const int32_t* lengths, const int32_t* perm, int32_t S_out, int32_t B,
                        int32_t* out_lengths, tzk_stream_t stream);
int tzk_permute_ids(const int64_t* ids, const int64_t* in_offsets, const int64_t* out_offsets,
                    const int32_t* perm, int32_t S_out, int32_t B, int64_t* out_ids,
                    tzk_stream_t stream);
/* the `weights` half of permute_2D_sparse_data: the per-sample weights of a weighted KJT, moved like its ids */
int tzk_permute_weights(const float* weights, const int64_t* in_offsets, const int64_t* out_offsets,
                        const int32_t* perm, int32_t S_out, int32_t B, float* out_weights, tzk_stream_t stream);

/* ---- K6: regroup  ([EXT] fbgemm::permute_pooled_embs / KeyedTensor.regroup_as_dict, called at
 * tzrec/modules/embedding.py:972-976; App. A.13) ------------------------------------------------------
 * Column gather-sum into ONE destination [rows, C]:
 *   out[row, c] = sum_{k in [col_start[c], col_start[c+1])} srcs[col_src[k]][row*src_ld[col_src[k]] + col_srccol[k]]
 * Forward regroup: one call per feature group, every output column has exactly one contributor.
 * Backward: destination = grad of a source KeyedTensor, contributors = the grads of every group that
 * copied the column (a feature may sit in several groups, e.g. DeepFM `fm` and `deep`); columns nobody
 * read get 0.  srcs_host / src_ld_host are HOST arrays (n_src <= 16) of device pointers / leading dims:
 * they travel as kernel parameters, so the call stays CUDA-graph capturable. */
int tzk_col_gather_sum(const float* const* srcs_host, const int64_t* src_ld_host, int32_t n_src,
                       const int32_t* col_start, const int32_t* col_src, const int32_t* col_srccol,
                       int32_t C, int64_t rows, float* out, int64_t ld_out, tzk_stream_t stream);

/* ---- K7: jagged -> padded dense and back  ([EXT] fbgemm::jagged_to_padded_dense via
 * JaggedTensor.to_padded_dense, tzrec/modules/embedding.py:1429,1480; App. A.14) ----------------------
 * out[b, t, 0:D] = values[offsets[b]+t] for t < min(len_b, T) else 0. */
int tzk_jagged_to_padded(const float* values, const int64_t* offsets, int32_t B, int32_t T, int32_t D,
                         float* out, tzk_stream_t stream);
/* backward: grad_values[offsets[b]+t] = grad_out[b,t] for t < min(len_b,T); rows beyond T get 0 */
int tzk_padded_to_jagged(const float* grad_out, const int64_t* offsets, int32_t B, int32_t T, int32_t D,
                         int64_t nnz, float* grad_values, tzk_stream_t stream);

/* ---- A7: factorization machine  (tzrec/modules/fm.py:28-42) ------------------------------------------
 * y[b,d] = 0.5 * ((sum_n x[b,n,d])^2 - sum_n x[b,n,d]^2);  x row b starts at x + b*ld_x, [N,D] dense. */
int tzk_fm_fwd(const float* x, int64_t ld_x, int64_t B, int32_t N, int32_t D, float* y, int64_t ld_y,
               tzk_stream_t stream);
/* dx[b,n,d] = dy[b,d] * (sum_n x[b,n,d] - x[b,n,d]) */
int tzk_fm_bwd(const float* x, int64_t ld_x, const float* dy, int64_t ld_dy, int64_t B, int32_t N,
               int32_t D, float* dx, int64_t ld_dx, tzk_stream_t stream);

/* ---- A9/A10: DLRM dot interaction  (tzrec/modules/interaction.py:80-91, concat glue
 * tzrec/models/dlrm.py:113-131) -----------------------------------------------------------------------
 * X_b = [dense[b] (optional, one row of D) ; sparse[b] (Ns rows of D)]  -> N = Ns + (dense != NULL)
 * out[b, 0:P]          = strict upper triangle of X_b X_b^T, row-major (triu_indices(N,N,1)), P=N(N-1)/2
 * out[b, P:P+D]        = dense[b]          (only if copy_dense  != 0)
 * out[b, .. : +Ns*D]   = sparse[b]         (only if copy_sparse != 0)
 * i.e. with both flags it emits the whole `final_mlp` input of DLRM in one pass. N <= 64, D <= 128.
 * p_pad in [0,3]: that many zero columns are inserted right after the P interaction terms, so that with
 * p_pad = (4 - P % 4) % 4 the dense and sparse blocks start on 16-B boundaries (128-bit stores, and 16-B aligned
 * rows for the GEMM that consumes the result; its weight gets matching zero columns). */
int tzk_dot_interact_fwd(const float* dense, int64_t ld_dense, const float* sparse, int64_t ld_sparse,
                         int64_t B, int32_t Ns, int32_t D, int32_t copy_dense, int32_t copy_sparse,
                         int32_t p_pad, float* out, int64_t ld_out, tzk_stream_t stream);
/* d_dense (nullable iff dense == NULL), d_sparse from d_out (same layout as `out`). */
int tzk_dot_interact_bwd(const float* dense, int64_t ld_dense, const float* sparse, int64_t ld_sparse,
                         const float* d_out, int64_t ld_dout, int64_t B, int32_t Ns, int32_t D,
                         int32_t copy_dense, int32_t copy_sparse, int32_t p_pad, float* d_dense,
                         int64_t ld_ddense, float* d_sparse, int64_t ld_dsparse, tzk_stream_t stream);
/* DLRM-Criteo (26 sparse features of D = 16 plus the bottom-MLP output, interaction output laid out
 * [351 pairs | 0 | dense 16 | sparse 416], 784 wide) followed by a 784 -> 64 layer: the backward of both at once.
 * d_dense [M,16] and d_sparse [M,416] from dz [M,64] (gradient of the layer's pre-activation) and its weight w [64, ld_w]
 * (columns 0..783 in the interaction's layout, ld_w >= 784); the layer's input gradient [M,784] is never written.
 * 3xTF32 like libtzk_gemm3x.so: the same bits as its input-gradient pass followed by tzk_dot_interact_bwd.  Row strides
 * multiples of 4 floats, every pointer 16-B aligned; wt_hi / wt_lo: [784, 64] scratch (the TF32 split of w^T).
 * (tzrec/models/dlrm.py:113-131 + tzrec/modules/mlp.py:20-84, backward) */
int tzk_interact_wide_bwd(const float* dz, int64_t ld_dz, const float* w, int64_t ld_w, const float* dense,
                          int64_t ld_dense, const float* sparse, int64_t ld_sparse, int64_t M, float* d_dense,
                          int64_t ld_ddense, float* d_sparse, int64_t ld_dsparse, float* wt_hi, float* wt_lo,
                          tzk_stream_t stream);
/* The same with dz read as dz * dz_scale[0] (a device scalar, e.g. the gradient reaching the loss), multiplied in
 * before the TF32 split: the bits of tzk_interact_wide_bwd on that product.  dz_scale NULL: no scaling. */
int tzk_interact_wide_bwd_scaled(const float* dz, int64_t ld_dz, const float* dz_scale, const float* w, int64_t ld_w,
                                 const float* dense, int64_t ld_dense, const float* sparse, int64_t ld_sparse, int64_t M,
                                 float* d_dense, int64_t ld_ddense, float* d_sparse, int64_t ld_dsparse, float* wt_hi,
                                 float* wt_lo, tzk_stream_t stream);
/* The forward of the same pair of layers: y [M,64] = relu(X w^T + bias) with X = [351 pairs | 0 | dense | sparse] the
 * interaction's output, and pairs [M,352] = X's first 352 columns (column 351 zero), which the weight gradient needs.
 * X itself is never written.  w [64, ld_w] in the interaction's column layout (ld_w >= 784), bias nullable; w_hi / w_lo:
 * [64, 784] scratch (the TF32 split of w).  Bit for bit tzk_dot_interact_fwd (p_pad = 1) followed by libtzk_gemm3x.so's
 * forward.  Row strides multiples of 4 floats, every pointer but bias 16-B aligned. */
int tzk_interact_wide_fwd(const float* dense, int64_t ld_dense, const float* sparse, int64_t ld_sparse, const float* w,
                          int64_t ld_w, const float* bias, int64_t M, float* y, int64_t ld_y, float* pairs,
                          int64_t ld_pairs, float* w_hi, float* w_lo, tzk_stream_t stream);
/* Weight gradient of the layer, dw [64, 784] = dz [M,64]^T X in X's column layout, with X read from pairs, dense and
 * sparse; bit for bit libtzk_gemm3x.so's tzk_wgrad3x on X with the same `slabs`.  partial: slabs * 896 * 64 floats of
 * scratch.  Row strides multiples of 4 floats, every pointer 16-B aligned. */
int tzk_interact_wide_wgrad(const float* dz, int64_t ld_dz, const float* pairs, int64_t ld_pairs, const float* dense,
                            int64_t ld_dense, const float* sparse, int64_t ld_sparse, int64_t M, int32_t slabs,
                            float* partial, float* dw, int64_t ld_dw, tzk_stream_t stream);
/* The same with dz read as dz * dz_scale[0], as tzk_interact_wide_bwd_scaled. */
int tzk_interact_wide_wgrad_scaled(const float* dz, int64_t ld_dz, const float* dz_scale, const float* pairs,
                                   int64_t ld_pairs, const float* dense, int64_t ld_dense, const float* sparse,
                                   int64_t ld_sparse, int64_t M, int32_t slabs, float* partial, float* dw,
                                   int64_t ld_dw, tzk_stream_t stream);

/* ---- dense-tower helpers (callers of the path: tzrec/modules/mlp.py:20-84, Perceptron = Linear -> ReLU) ----
 * The tower GEMMs stay library calls; these fuse the element-wise passes around them.
 *   tzk_bias_act        : y[r, 0:N] = act(y[r, 0:N] + bias)            (in place; bias nullable; relu 0/1)
 *   tzk_act_bwd_colsum  : dz = dy * (y > 0) (or dy if !relu; dz nullable), colsum[c] = sum_r dz[r,c]
 *                         deterministic two-stage column sum; N must divide 256. */
int tzk_bias_act(float* y, int64_t ld_y, const float* bias, int64_t M, int32_t N, int32_t relu,
                 tzk_stream_t stream);
size_t tzk_act_bwd_colsum_workspace_bytes(int64_t M, int32_t N);
int tzk_act_bwd_colsum(const float* dy, int64_t ld_dy, const float* y, int64_t ld_y, int64_t M, int32_t N,
                       int32_t relu, float* dz, int64_t ld_dz, float* colsum, void* workspace,
                       size_t workspace_bytes, tzk_stream_t stream);

/* ---- narrow fully-connected layers (K, N <= 64) and the BCE head — the layers either side of the interaction
 * in every rank model (tzrec/modules/mlp.py:20-84; DLRM bottom MLP 13->64->16 and the 64->32->1 end of its final
 * MLP, tzrec/models/dlrm.py:60-99; BCEWithLogitsLoss tzrec/models/rank_model.py:190-216).  One launch per layer
 * forward, one (+ a fixed-order partial reduction) backward; fp32 FFMA in ascending-k order.
 *   fwd : y[M,N]  = act(x[M,K] @ w[N,K]^T + bias)                      (bias nullable; relu 0/1)
 *   bwd : dz = dy * (y > 0) (or dy if !relu);  dx[M,K] = dz @ w (dx nullable);  dw[N,K] = dz^T @ x;
 *         db[N] = column sums of dz (db nullable).  Deterministic.
 *   bce : loss[0] = mean_i( max(z,0) - z*t + log1p(exp(-|z|)) ),  dlogits[i] = (sigmoid(z_i) - t_i) / M
 *         (dlogits nullable). */
int tzk_small_linear_fwd(const float* x, int64_t ld_x, const float* w, const float* bias, int64_t M, int32_t K,
                         int32_t N, int32_t relu, float* y, int64_t ld_y, tzk_stream_t stream);
size_t tzk_small_linear_bwd_workspace_bytes(int64_t M, int32_t K, int32_t N);
int tzk_small_linear_bwd(const float* x, int64_t ld_x, const float* w, const float* y, int64_t ld_y,
                         const float* dy, int64_t ld_dy, int64_t M, int32_t K, int32_t N, int32_t relu, float* dx,
                         int64_t ld_dx, float* dw, float* db, void* workspace, size_t workspace_bytes,
                         tzk_stream_t stream);
size_t tzk_bce_logits_workspace_bytes(int64_t M);

/* ---- the tower tail in one pass, forward AND backward: last Perceptron of the final MLP (K -> N with ReLU,
 * tzrec/modules/mlp.py:20-84), output Linear(N, 1) and mean BCE-with-logits on the label (tzrec/models/rank_model.py:
 * 133-179, 181-262).  h = relu(y1 @ w1^T + b1); logits = h @ w2^T + b2; loss as tzk_bce_logits; and d loss / d ... :
 * dy1 [M, K] and out = [dW1 (N x K, row-major) | db1 (N) | dw2 (N) | db2 (1) | loss (1)].  K, N <= 64; b1, b2 nullable.
 * Deterministic (fixed-order folds).  Replaces 18 launches of the unfused chain on DLRM-Criteo (64 -> 32 -> 1).
 * colsum nullable.  Given (y1 the output of a ReLU layer), dy1 receives dz = dy1 * (y1 > 0) instead, the gradient of
 * that layer's pre-activation, and colsum [K] its column sums (at K = 64 the bits of tzk_act_bwd_colsum on dy1, y1). */
size_t tzk_tower_tail_bce_workspace_bytes(int64_t M, int32_t K, int32_t N);
int tzk_tower_tail_bce(const float* y1, int64_t ld_y, const float* w1, const float* b1, const float* w2, const float* b2,
                       const float* labels, int64_t M, int32_t K, int32_t N, float* logits, float* dy1, int64_t ld_dy,
                       float* colsum, float* out, void* workspace, size_t workspace_bytes, tzk_stream_t stream);
int tzk_bce_logits_fwd_bwd(const float* logits, const float* labels, int64_t M, float* loss, float* dlogits,
                           void* workspace, size_t workspace_bytes, tzk_stream_t stream);

/* ---- DIN target attention over jagged sequence rows (tzrec/modules/sequence.py:65-128 without the padded
 * [B, T, Ds] tensor of tzrec/modules/embedding.py:1466-1480; SURVEY §8f N3).  seq [N, Ds]: the un-pooled lookup's rows,
 * sample b owns rows offsets[b] .. offsets[b+1]; query [B, Dq] (row stride ld_q), Dq <= Ds (zero-padded to Ds).
 *   din_attn_input_fwd : out[n, :] = [q_b | k_n | q_b - k_n | q_b * k_n]            ([N, 4 * Ds])
 *   din_attn_input_bwd : d_seq[n] = g2 - g3 + g4 * q_b, d_query[b] = sum_n (g1 + g3 + g4 * k_n)   (rows in order)
 *   jagged_softmax_wsum_fwd : p = softmax(scores[first min(len, max_len) rows of b]) (max_len <= 0: all), probs[n]
 *                             (0 beyond max_len), out[b] = sum_n p_n k_n; a sample without rows gives zeros
 *   jagged_softmax_wsum_bwd : d_scores[n] = p_n (<d_out_b, k_n> - sum_m p_m <d_out_b, k_m>), d_seq[n] = p_n d_out_b */
int tzk_din_attn_input_fwd(const float* query, int64_t ld_q, int32_t Dq, const float* seq, const int64_t* offsets,
                           int32_t B, int32_t Ds, int64_t N, float* out, tzk_stream_t stream);
int tzk_din_attn_input_bwd(const float* d_in, const float* query, int64_t ld_q, int32_t Dq, const float* seq,
                           const int64_t* offsets, int32_t B, int32_t Ds, int64_t N, float* d_query, float* d_seq,
                           tzk_stream_t stream);
int tzk_jagged_softmax_wsum_fwd(const float* scores, const float* seq, const int64_t* offsets, int32_t B, int32_t Ds,
                                int32_t max_len, int64_t N, float* probs, float* out, tzk_stream_t stream);
int tzk_jagged_softmax_wsum_bwd(const float* d_out, const float* probs, const float* seq, const int64_t* offsets,
                                int32_t B, int32_t Ds, int32_t max_len, int64_t N, float* d_scores, float* d_seq,
                                tzk_stream_t stream);

/* ---- sharded sparse step over peer memory (NVSwitch domain; replaces the KJT / pooled-embedding / sequence-embedding
 * all-to-alls and the reduce-scatter of torchrec's ShardedEmbeddingBagCollection / ShardedEmbeddingCollection and the DDP
 * all-reduce of the dense gradients: SURVEY.md §2.3 C1-C5, App. A.5-A.8, reached from tzrec/main.py:799).  `*_ptrs`
 * are HOST arrays [W] of device addresses: rank r's symmetric buffer as mapped in the calling process (W <= 16).
 *   peer_pooled_gather_fwd : the requester's gather reads each row from the owning rank's arena (owner = feat_owner +
 *                            id / feat_block, as tzk_bucketize_rw) and pools locally; rf_w_off[r * F + f] = arena
 *                            offset (elements) of feature f's table on rank r; other arrays as tzk_pooled_gather_fwd.
 *   peer_seq_gather_fwd    : the same for un-pooled lookups: out[l, :] = row of ids[l] (all features share D).
 *   peer_barrier           : one CTA; flag[src] on every rank = epoch, st.release.sys / ld.acquire.sys; `epoch` is a
 *                            device counter (graph-replayable).  Every rank must call it the same number of times per
 *                            (pad_ptrs, epoch) pair; barrier sites that can overlap in time use different pairs.
 *   peer_bucketize         : source side of the backward.  Stable multi-split of the local ids by destination into
 *                            this rank's wire buffers: destination r's entries start at r * cap, in (feature, bag,
 *                            position) order; wire_key = rf_key_base[r * F + f] + owner-local row (the owner's
 *                            linearised sort key), wire_idx = bag index f * B + b (pooled) or id position (sequence);
 *                            counts[r] = ids for r (clamped to cap), counts[W] = 1 if any destination overflowed.
 *   peer_publish_grad      : dst[b, col_f : col_f + D_f] = grad[b, ...] (/ bag length for MEAN features).
 *   peer_allreduce_mean    : out[i] = (src_0[i] + ... + src_{W-1}[i]) / W, summed in rank order.
 *   fused_bwd_sort_peer / fused_bwd_apply_peer : owner side of the backward — tzk_fused_bwd_sort / _apply over the
 *                            W * cap wire slots of this rank: keys pulled from the sources' wire buffers, gradient
 *                            slices read from the sources' published gradients; idx_span > every wire_idx.
 * Return 0, or 1 bad argument / 3 launch failure. */
int tzk_peer_pooled_gather_fwd(const uint64_t* table_ptrs, const int64_t* rf_w_off, const int64_t* feat_rows,
                               const int64_t* feat_block, const int32_t* feat_owner, const int32_t* feat_dim,
                               const int32_t* feat_col, const int32_t* feat_pool, const int64_t* ids,
                               const int64_t* offsets, int32_t F, int32_t B, int32_t W, int32_t max_dim, float* out,
                               int64_t ld_out, const float* mirror, const int64_t* feat_mirror_off, tzk_stream_t stream);
/* the same lookup for the features listed in feat_sel [n_sel] only (device int32 indices into the F descriptors; only their
 * output columns are written): complementary lists on two streams overlap the mirrored half with the NVLink half */
int tzk_peer_pooled_gather_fwd_sel(const uint64_t* table_ptrs, const int64_t* rf_w_off, const int64_t* feat_rows,
                                   const int64_t* feat_block, const int32_t* feat_owner, const int32_t* feat_dim,
                                   const int32_t* feat_col, const int32_t* feat_pool, const int64_t* ids,
                                   const int64_t* offsets, int32_t F, int32_t B, int32_t W, int32_t max_dim, float* out,
                                   int64_t ld_out, const float* mirror, const int64_t* feat_mirror_off,
                                   const int32_t* feat_sel, int32_t n_sel, tzk_stream_t stream);
int tzk_peer_seq_gather_fwd(const uint64_t* table_ptrs, const int64_t* rf_w_off, const int64_t* feat_rows,
                            const int64_t* feat_block, const int32_t* feat_owner, const int64_t* ids,
                            const int64_t* offsets, int32_t F, int32_t B, int32_t W, int32_t D, int64_t nnz, float* out,
                            const float* mirror, const int64_t* feat_mirror_off, tzk_stream_t stream);
/* mirror / feat_mirror_off (both may be NULL): features with feat_mirror_off[f] >= 0 read row id at
 * mirror[feat_mirror_off[f] + id * D_f] — this rank's per-step copy of the WHOLE (small) table, refreshed by
 * peer_mirror_refresh from n_seg contiguous pieces (rank seg_rank[s], arena offset seg_src[s], mirror offset seg_dst[s],
 * seg_n[s] floats; device arrays). */
int tzk_peer_mirror_refresh(const uint64_t* table_ptrs, int32_t W, const int32_t* seg_rank, const int64_t* seg_src,
                            const int64_t* seg_dst, const int64_t* seg_n, int32_t n_seg, float* mirror,
                            tzk_stream_t stream);
int tzk_peer_barrier(const uint64_t* pad_ptrs, int32_t me, int32_t W, uint32_t* epoch, tzk_stream_t stream);
size_t tzk_peer_bucketize_workspace_bytes(int32_t F, int32_t B, int32_t W);
int tzk_peer_bucketize(const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B, int32_t W,
                       const int64_t* feat_block, const int32_t* feat_owner, const int64_t* feat_rows,
                       const int64_t* rf_key_base, int32_t pooled, int64_t cap, int64_t* wire_key, int32_t* wire_idx,
                       int32_t* counts, void* workspace, size_t workspace_bytes, tzk_stream_t stream);
int tzk_peer_publish_grad(const float* grad, int64_t ld_grad, const int32_t* feat_col, const int32_t* feat_dim,
                          const int32_t* feat_pool, const int64_t* offsets, int32_t F, int32_t B, float* dst,
                          int64_t ld_dst, tzk_stream_t stream);
/* peer_push_grad: wire slot (dest r, j) of this rank -> row me * cap + j of rank r's receive buffer [W * cap, D]
 * (coalesced NVLink writes; MEAN bags divided by their length); the owner then sorts with idx_span = 0 ("slot mode":
 * the sorted value is the receive-buffer row) and runs the plain sequence-layout tzk_fused_bwd_apply on that buffer. */
int tzk_peer_push_grad(const uint64_t* recv_ptrs, const float* grad, int64_t ld_grad, const int32_t* feat_col,
                       const int32_t* feat_pool, const int64_t* offsets, const int32_t* wire_idx, const int32_t* counts,
                       int32_t me, int32_t W, int64_t cap, int32_t B, int32_t D, int32_t pooled, tzk_stream_t stream);
int tzk_peer_allreduce_mean(const uint64_t* src_ptrs, int32_t W, int64_t n, float* out, tzk_stream_t stream);
/* Small tables (the mirrored ones): every rank reduces its own batch's gradients per row into a dense buffer
 * psum [R_small, dim] + flags [R_small] (tzk_fused_bwd_apply_ex with TZK_OPT_ACCUM_OUT over a layout whose w_off / key_base
 * address that buffer); the owner of a row then adds the W partial sums in rank order (sequential NVLink reads) and
 * applies one update: tzk_peer_small_update.  `tabs`: device array of n_tabs records
 * { int64 kb_small, start, w_off, psum_off, key_base; int32 first, n_local, dim, pad } — per small table: its first key
 * in the small key space, this rank's first global row, the shard's arena offset, the table's offset in psum, the
 * shard's local key base, the prefix sum of local rows, the local row count, the dim.  total_rows = sum of n_local. */
int tzk_peer_small_update(const tzk_opt_args* opt, const uint64_t* psum_ptrs, const uint64_t* flag_ptrs, int32_t W,
                          const void* tabs, int32_t n_tabs, int32_t total_rows, int32_t max_dim, float* weights,
                          tzk_stream_t stream);
int tzk_fused_bwd_sort_peer(const uint64_t* key_ptrs, const uint64_t* idx_ptrs, const uint64_t* count_ptrs, int32_t me,
                            int32_t W, int64_t cap, int32_t idx_span, int64_t total_keys, int32_t max_dim,
                            int32_t* overflow, void* workspace, size_t workspace_bytes, tzk_stream_t stream);
int tzk_fused_bwd_apply_peer(const tzk_opt_args* opt, int32_t pooled, const uint64_t* grad_ptrs, int64_t ld_grad,
                             const int64_t* feat_w_off, const int64_t* feat_rows, const int32_t* feat_dim,
                             const int32_t* feat_col, const int32_t* feat_pool, const int64_t* feat_key_base, int32_t F,
                             int32_t B, int32_t me, int32_t W, int64_t cap, int32_t idx_span, int64_t total_keys,
                             int32_t max_dim, int32_t vec_ok, float* weights, float grad_scale, void* workspace,
                             size_t workspace_bytes, tzk_stream_t stream);

/* ---- weighted bags on the peer step ([EXT] torchrec's sharded lookup passes features.weights_or_none() to the TBE on
 * every sharding type).  The per-sample weights never leave the sample's rank: its gather pools w[l] * row, its
 * bucketize records the weight of every wire slot in a LOCAL buffer, its push sends w * g (/ L).  The owner's update is
 * the unweighted one (grad_scale 1/W).  Pooled layouts, push transport only; the pull transport
 * (tzk_fused_bwd_apply_peer) and tzk_peer_small_update keep requiring opt->per_sample_weights == NULL.
 *   peer_pooled_gather_fwd_weighted : tzk_peer_pooled_gather_fwd / _sel (feat_sel NULL: every feature) with the
 *                            arithmetic of tzk_pooled_gather_fwd_weighted: acc = w[l0] * row, then fmaf(w[l], row, acc)
 *                            in list order, MEAN * 1/L — the same bits as the unsharded weighted lookup.
 *   peer_bucketize_weighted: tzk_peer_bucketize (pooled != 0) + wire_w[r * cap + slot] = per_sample_weights[l], wire_w a
 *                            local float buffer of W * cap entries.
 *   peer_push_grad_weighted: tzk_peer_push_grad (pooled != 0) with every slice scaled by ((1/L for MEAN) * wire_w[s]). */
int tzk_peer_pooled_gather_fwd_weighted(const uint64_t* table_ptrs, const int64_t* rf_w_off, const int64_t* feat_rows,
                                        const int64_t* feat_block, const int32_t* feat_owner, const int32_t* feat_dim,
                                        const int32_t* feat_col, const int32_t* feat_pool, const int64_t* ids,
                                        const int64_t* offsets, int32_t F, int32_t B, int32_t W, int32_t max_dim,
                                        float* out, int64_t ld_out, const float* mirror, const int64_t* feat_mirror_off,
                                        const float* per_sample_weights, const int32_t* feat_sel, int32_t n_sel,
                                        tzk_stream_t stream);
int tzk_peer_bucketize_weighted(const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B, int32_t W,
                                const int64_t* feat_block, const int32_t* feat_owner, const int64_t* feat_rows,
                                const int64_t* rf_key_base, int32_t pooled, int64_t cap, int64_t* wire_key,
                                int32_t* wire_idx, int32_t* counts, void* workspace, size_t workspace_bytes,
                                const float* per_sample_weights, float* wire_w, tzk_stream_t stream);
int tzk_peer_push_grad_weighted(const uint64_t* recv_ptrs, const float* grad, int64_t ld_grad, const int32_t* feat_col,
                                const int32_t* feat_pool, const int64_t* offsets, const int32_t* wire_idx,
                                const int32_t* counts, int32_t me, int32_t W, int64_t cap, int32_t B, int32_t D,
                                int32_t pooled, const float* wire_w, tzk_stream_t stream);

/* ---- DLRM-Criteo interaction in BF16 (train_config.mixed_precision "BF16"; csrc/tzk_interact_bf16.cuh).  bf16 values
 * cross the ABI as their 16-bit patterns.  N = 27 rows of 16 (dense + 26 sparse features); the row
 * X = [351 pairs | 0 | 16 dense | 416 sparse] is 784 bf16, the reference's 783 columns with one zero after the pairs.
 *   fwd_bf16: pairs = bf16_rn(F F^T) (products exact, fp32 accumulation, mma.sync m16n8k16) over F = [dense ; bf16_rn(sparse)];
 *             the copied columns are dense as it is and bf16_rn(sparse).
 *   bwd_bf16: from dX (bf16), with G the pair gradient in the upper triangle and g1 = bf16_rn(G F), g2 = bf16_rn(G^T F),
 *             s = fp32(g1 + g2): d_dense = bf16_rn(bf16_rn(s) + dX_dense), d_sparse = s + dX_sparse (fp32) — autograd's
 *             rounding points under torch.autocast(dtype=torch.bfloat16).
 * Rows: dense / d_dense 8-B aligned with ld a multiple of 4, sparse / d_sparse 16-B aligned with ld a multiple of 4,
 * X / dX 16-B aligned with ld a multiple of 8; anything else is rejected. */
int tzk_dot_interact27_fwd_bf16(const uint16_t* dense, int64_t ld_dense, const float* sparse, int64_t ld_sparse, int64_t B,
                                uint16_t* out, int64_t ld_out, tzk_stream_t stream);
int tzk_dot_interact27_bwd_bf16(const uint16_t* d_out, int64_t ld_dout, const uint16_t* dense, int64_t ld_dense,
                                const float* sparse, int64_t ld_sparse, int64_t B, uint16_t* d_dense, int64_t ld_ddense,
                                float* d_sparse, int64_t ld_dsparse, tzk_stream_t stream);

/* ---- evaluation metrics (csrc/tzk_metrics.cuh) --------------------------------------------------------------------
 * binned_auc_update: the update of torchmetrics.AUROC(task="binary", thresholds=T) (tzrec/models/rank_model.py:392-398,
 * `_binary_precision_recall_curve_update_vectorized`) as a histogram.  For i < n with label y in {0, 1} and p in [0, 1]:
 *     counts[bin(p) * 2 + y] += 1,  bin(p) = #{k < T : p >= thresholds[k]}  (0..T; thresholds nondecreasing);
 * any other sample (label outside {0, 1}, p NaN or outside [0, 1]) adds 1 to *invalid instead.  counts is int64
 * [(T + 1) * 2] and is accumulated into, never cleared.  preds: pred_dtype 0 = fp32, 1 = bf16 (16-bit patterns);
 * labels: label_dtype 0 = fp32, 1 = int64.  Deterministic (integer atomics).  n = 0 launches nothing. */
int tzk_binned_auc_update(const void* preds, int32_t pred_dtype, const void* labels, int32_t label_dtype, int64_t n,
                          const float* thresholds, int32_t T, int64_t* counts, int64_t* invalid, tzk_stream_t stream);

/* ---- FP16 tables on the peer step: every rank's arena (table_ptrs) and the local mirror hold IEEE halfs; everything
 * else — outputs, gradients on the wire, receive buffers, published gradients, partial sums, optimizer state — stays
 * fp32.  Arguments as in the fp32 entry points above; dims must be multiples of 4 (rows 8-B aligned).
 *   peer_pooled_gather_fwd_f16 / _sel_f16 / _weighted_f16, peer_seq_gather_fwd_f16: every row (owner arena or mirror)
 *                            is read with a coherent 8-B load and widened exactly; pooling as tzk_pooled_gather_fwd_f16,
 *                            tzk_pooled_gather_fwd_weighted (weights_f16 = 1) and tzk_seq_gather_fwd_f16 — the same bits.
 *   peer_mirror_refresh_f16: segments counted in halfs (multiples of 4), copied bit for bit in 8-B vectors.
 * The owner-side updates take a half arena through tzk_opt_args.weights_f16: tzk_fused_bwd_apply_peer (pull transport),
 * tzk_fused_bwd_apply_ex over the receive buffer (push) and tzk_peer_small_update widen the row, update in fp32 and
 * round back to nearest even. */
int tzk_peer_pooled_gather_fwd_f16(const uint64_t* table_ptrs, const int64_t* rf_w_off, const int64_t* feat_rows,
                                   const int64_t* feat_block, const int32_t* feat_owner, const int32_t* feat_dim,
                                   const int32_t* feat_col, const int32_t* feat_pool, const int64_t* ids,
                                   const int64_t* offsets, int32_t F, int32_t B, int32_t W, int32_t max_dim, float* out,
                                   int64_t ld_out, const void* mirror, const int64_t* feat_mirror_off,
                                   tzk_stream_t stream);
int tzk_peer_pooled_gather_fwd_sel_f16(const uint64_t* table_ptrs, const int64_t* rf_w_off, const int64_t* feat_rows,
                                       const int64_t* feat_block, const int32_t* feat_owner, const int32_t* feat_dim,
                                       const int32_t* feat_col, const int32_t* feat_pool, const int64_t* ids,
                                       const int64_t* offsets, int32_t F, int32_t B, int32_t W, int32_t max_dim,
                                       float* out, int64_t ld_out, const void* mirror, const int64_t* feat_mirror_off,
                                       const int32_t* feat_sel, int32_t n_sel, tzk_stream_t stream);
int tzk_peer_pooled_gather_fwd_weighted_f16(const uint64_t* table_ptrs, const int64_t* rf_w_off,
                                            const int64_t* feat_rows, const int64_t* feat_block,
                                            const int32_t* feat_owner, const int32_t* feat_dim, const int32_t* feat_col,
                                            const int32_t* feat_pool, const int64_t* ids, const int64_t* offsets,
                                            int32_t F, int32_t B, int32_t W, int32_t max_dim, float* out, int64_t ld_out,
                                            const void* mirror, const int64_t* feat_mirror_off,
                                            const float* per_sample_weights, const int32_t* feat_sel, int32_t n_sel,
                                            tzk_stream_t stream);
int tzk_peer_seq_gather_fwd_f16(const uint64_t* table_ptrs, const int64_t* rf_w_off, const int64_t* feat_rows,
                                const int64_t* feat_block, const int32_t* feat_owner, const int64_t* ids,
                                const int64_t* offsets, int32_t F, int32_t B, int32_t W, int32_t D, int64_t nnz,
                                float* out, const void* mirror, const int64_t* feat_mirror_off, tzk_stream_t stream);
int tzk_peer_mirror_refresh_f16(const uint64_t* table_ptrs, int32_t W, const int32_t* seg_rank, const int64_t* seg_src,
                                const int64_t* seg_dst, const int64_t* seg_n, int32_t n_seg, void* mirror,
                                tzk_stream_t stream);

/* ---- WuKong layer (tzrec/modules/interaction.py:236-378) around its dense FMB MLP, X [B, n, d] fp32 row-major, m = f + l.
 * Shapes: n <= 64, d in {4, 8, 16, 32}, k <= 32, f, l >= 1, f + l <= 64.  All weights row-major as the reference
 * stores them: w_fmb [n, k], w_lcb [n, l], w_res [n, m] (NULL: identity residual, needs n == m); gamma / beta of the FMB
 * norm [n * k], of the output norm [d].  LayerNorm eps 1e-5.  Everything is fp32 FFMA.  `grid` CTAs walk the samples
 * (rows) grid-stride; weight / gamma / beta gradients are per-CTA partial sums (`partials`, grid x P floats) reduced in
 * CTA order into `dparams`: deterministic for a given grid, no float atomics.
 *   mix_fwd: ln_f [B, n * k] = LayerNorm(X (X^T w_fmb)) with affine, stats [B, 2] = (mean, rstd);
 *            base [B, m, d] = residual (w_res^T X or X) with w_lcb^T X added to rows >= f.
 *   mix_bwd: d_ln_f [B, n * k], d_base [B, m, d] -> dx [B, n, d] and dparams (P floats) =
 *            dw_fmb [n k] | dw_lcb [n l] | dw_res [n m] (w_res only) | dgamma [n k] | dbeta [n k].  F is recomputed.
 *   out_fwd: y [B, m, d] = LayerNorm_d(z) with affine, z = fmb_out [B, f * d] + base on rows < f, base on the rest;
 *            stats [B, m, 2].
 *   out_bwd: dy -> d_fmb_out [B, f * d], d_base [B, m, d], dparams (2 d floats) = dgamma | dbeta. */
int tzk_wukong_mix_fwd(const float* x, const float* w_fmb, const float* gamma, const float* beta, const float* w_lcb,
                       const float* w_res, int64_t B, int32_t n, int32_t d, int32_t k, int32_t f, int32_t l,
                       int32_t grid, float* ln_f, float* stats, float* base, tzk_stream_t stream);
int tzk_wukong_mix_bwd(const float* x, const float* w_fmb, const float* gamma, const float* w_lcb, const float* w_res,
                       const float* stats, const float* d_ln_f, const float* d_base, int64_t B, int32_t n, int32_t d,
                       int32_t k, int32_t f, int32_t l, int32_t grid, float* dx, float* partials, float* dparams,
                       tzk_stream_t stream);
int tzk_wukong_out_fwd(const float* fmb_out, const float* base, const float* gamma, const float* beta, int64_t B,
                       int32_t d, int32_t f, int32_t l, int32_t grid, float* y, float* stats, tzk_stream_t stream);
int tzk_wukong_out_bwd(const float* fmb_out, const float* base, const float* gamma, const float* stats,
                       const float* dy, int64_t B, int32_t d, int32_t f, int32_t l, int32_t grid, float* d_fmb_out,
                       float* d_base, float* partials, float* dparams, tzk_stream_t stream);

/* ---- MaskNet's parallel mask blocks (tzrec/modules/masknet.py:77-85, 142-155) around their GEMMs.  nb blocks, input
 * width E, FFN width H; Ep = E rounded up to a multiple of 4 is the row pitch of every [B, nb Ep] operand, so the GEMMs
 * between these stages run on 16-B aligned rows.  Shapes: pad4(E) <= 1024, 4 <= H <= 1024 with H % 4 == 0,
 * 1 <= nb <= 8.  fp32 row-major; LayerNorm eps 1e-5; fp32 FFMA.  `grid` CTAs walk the samples grid-stride; batch sums
 * (bias / gamma / beta gradients) are per-CTA partials (`partials`) reduced in CTA order into `dparams`: deterministic
 * for a given grid, no float atomics.
 *   mask_fwd: e [B, lde] (first E columns), m [B, nb Ep] (the mask generators' second GEMM, no bias), b2 [nb E],
 *             gamma / beta [E] of ln_emb -> v [B, nb Ep] = LN(e) * (m_i + b2_i) per block (pad columns 0),
 *             stats [B, 2] = (mean, rstd).  Replaces ln_emb, the bias add and `feature_input * weights` (:80, :144).
 *   mask_bwd: dv [B, nb Ep] -> dm [B, nb Ep] = dv_i * LN(e), de [B, Ep] = LayerNorm backward of
 *             sum_i dv_i * (m_i + b2_i) (pad columns 0), dparams ((nb + 2) E floats) = db2 [nb E] | dgamma | dbeta.
 *             partials: grid x (nb + 2) E floats.
 *   ffn_fwd:  z [B, nb H] (each block's ffn.0 GEMM, no bias), b3 / gamma / beta [nb H] -> y [B, nb H] =
 *             ReLU(LN_H(z_i + b3_i)) in block i's column slot (the concat at :145-151), stats [B, nb, 2].
 *             Replaces ffn's bias add, LayerNorm and ReLU (:68-72, :82).
 *   ffn_bwd:  dy [B, nb H] -> dz [B, nb H], dparams (nb x 3 H floats) = per block dgamma | dbeta | db3.
 *             partials: nb x grid x 3 H floats. */
int tzk_masknet_mask_fwd(const float* e, int32_t lde, const float* m, const float* b2, const float* gamma,
                         const float* beta, int64_t B, int32_t E, int32_t nb, int32_t grid, float* v, float* stats,
                         tzk_stream_t stream);
int tzk_masknet_mask_bwd(const float* e, int32_t lde, const float* m, const float* b2, const float* gamma,
                         const float* beta, const float* stats, const float* dv, int64_t B, int32_t E, int32_t nb,
                         int32_t grid, float* dm, float* de, float* partials, float* dparams, tzk_stream_t stream);
int tzk_masknet_ffn_fwd(const float* z, const float* b3, const float* gamma, const float* beta, int64_t B, int32_t H,
                        int32_t nb, int32_t grid, float* y, float* stats, tzk_stream_t stream);
int tzk_masknet_ffn_bwd(const float* z, const float* b3, const float* gamma, const float* beta, const float* stats,
                        const float* dy, int64_t B, int32_t H, int32_t nb, int32_t grid, float* dz, float* partials,
                        float* dparams, tzk_stream_t stream);

/* ---- PLE: the gates of one extraction layer (tzrec/modules/extraction_net.py:93-105 `_gate_forward`, called at
 * :120-133), all of them in one launch each way.  n_gates gates (the T task gates, then the shared gate when the layer
 * is not the last); gate g reads input gate_input[g] (one of n_inputs distinct [B, in_dim[i]] tensors) and mixes the
 * gate_num_experts[g] experts listed in gate_experts[g] (indices into the n_experts [B, H] expert outputs, in the
 * reference's stack order).  Gate weights [E_g, K_g] and biases [E_g] of nn.Linear.  fp32 row-major, fp32 FFMA.
 * Cover: 1 <= n_gates <= 9, n_experts <= 64, 1 <= E_g <= 32 distinct experts, 1 <= H <= 1024, 1 <= K_i <= 1024, and
 * sum_g E_g K_g <= 20480 floats (the weights stay in shared memory; the backward holds them and their gradient).
 * The description travels by value as a kernel parameter (no host-to-device copy: graph-capturable); its device
 * pointers are read when the call is made.
 *   gate_fwd: -> y [n_gates, B, H] (y_g = sum_e softmax(x_g W_g^T + b_g)_e expert_e), p [B, sum E_g] (the softmax,
 *             gate g at column sum_{g' < g} E_g').
 *   gate_bwd: dy [n_gates, B, H] -> d_experts [n_experts, B, H] (written once per element, the gates summed in
 *             order), d_inputs[i] [B, K_i] (sum over the gates reading input i), dparams = dW_0 | dW_1 | ... | db_0 |
 *             db_1 | ... (sum_g E_g K_g + sum_g E_g floats): per-CTA partials (grid rows of that size) reduced in CTA
 *             order, no float atomics.
 *   gate_smem_bytes: dynamic shared memory of one CTA of the forward (backward = 0) or the backward (1) launch; 0 when
 *             the description is outside the cover.  Needs no GPU. */
#define TZK_PLE_MAX_GATES 9
#define TZK_PLE_MAX_EXPERTS 64
#define TZK_PLE_MAX_GATE_EXPERTS 32
typedef struct tzk_ple_gate_args {
  int64_t B;
  int32_t H, n_experts, n_inputs, n_gates;
  int32_t in_dim[TZK_PLE_MAX_GATES];
  int32_t gate_input[TZK_PLE_MAX_GATES];
  int32_t gate_num_experts[TZK_PLE_MAX_GATES];
  uint8_t gate_experts[TZK_PLE_MAX_GATES][TZK_PLE_MAX_GATE_EXPERTS];
  const float* experts[TZK_PLE_MAX_EXPERTS];
  const float* inputs[TZK_PLE_MAX_GATES];
  const float* weight[TZK_PLE_MAX_GATES];
  const float* bias[TZK_PLE_MAX_GATES];
  float* d_inputs[TZK_PLE_MAX_GATES]; /* gate_bwd only */
} tzk_ple_gate_args;
int64_t tzk_ple_gate_smem_bytes(const tzk_ple_gate_args* args_host, int32_t backward);
int tzk_ple_gate_fwd(const tzk_ple_gate_args* args_host, int32_t grid, float* y, float* p, tzk_stream_t stream);
int tzk_ple_gate_bwd(const tzk_ple_gate_args* args_host, const float* p, const float* dy, int32_t grid,
                     float* d_experts, float* partials, float* dparams, tzk_stream_t stream);

/* ---- PEPNet: the gate-neural-unit product (tzrec/modules/personalized_net.py: GateNU.forward :50-59 scaling
 * EPNet.forward :90-110 and the body of PPNet.forward's loop :187-195), up to 8 segments in one launch each way.
 * Segment s is [B, N] (4 <= N <= 1024, N % 4 == 0, row pitches multiples of 4 floats, 16-B aligned pointers):
 *   gate_fwd: y = act(x + bx) * gamma sigmoid(z + bz)       act: identity or ReLU; bx may be NULL (no bias)
 *   gate_bwd: dy -> dx = dy * gamma s * act'(x + bx), dz = dy * act(x + bx) * gamma s (1 - s), s = sigmoid(z + bz)
 *             recomputed from x and z; dparams = dbx_0 | dbz_0 | dbx_1 | dbz_1 | ... (2 N_s floats per segment) as
 *             per-CTA partials (grid rows of that size) reduced in CTA order, no float atomics.
 * x, z, y, dy, dx, dz use the pitches ldx (x, dx), ldz (z, dz) and ldy (y, dy).  fp32.  The description travels by
 * value as a kernel parameter (no host-to-device copy: graph-capturable). */
#define TZK_PEPNET_MAX_SEGS 8
#define TZK_PEPNET_IDENTITY 0
#define TZK_PEPNET_RELU 1
typedef struct tzk_pepnet_seg {
  const float* x;
  const float* bx;
  const float* z;
  const float* bz;
  float* y;        /* gate_fwd only */
  const float* dy; /* gate_bwd only */
  float* dx;       /* gate_bwd only */
  float* dz;       /* gate_bwd only */
  int64_t ldx, ldz, ldy;
  int32_t N, act;
  float gamma;
  int32_t pad_;
} tzk_pepnet_seg;
typedef struct tzk_pepnet_gate_args {
  int64_t B;
  int32_t n_segs, pad_;
  tzk_pepnet_seg seg[TZK_PEPNET_MAX_SEGS];
} tzk_pepnet_gate_args;
int tzk_pepnet_gate_fwd(const tzk_pepnet_gate_args* args_host, int32_t grid, tzk_stream_t stream);
int tzk_pepnet_gate_bwd(const tzk_pepnet_gate_args* args_host, int32_t grid, float* partials, float* dparams,
                        tzk_stream_t stream);

/* ---- JRC loss (tzrec/loss/jrc_loss.py) and its gradient in one call, O(B) memory.  logits [B, 2] with row pitch
 * ld >= 2, labels [B] fp32 (0 or 1), session_ids [B] int64 (ids in [0, 2^key_bits); key_bits 64 for any id),
 * weights [B] or NULL.  loss[0] = (1/B) sum_i w_i (alpha ce_i + (1 - alpha) ge_i) with w_i = 1 when weights is NULL;
 * dlogits [B, 2] contiguous = d loss / d logits.  NaN loss (finite gradient) for B = 0 and, with weights NULL, for a
 * batch without a positive or a negative; a label outside {0, 1} gives a NaN loss and gradient row.  Deterministic
 * (no float atomics), no host synchronisation: graph-capturable. */
size_t tzk_jrc_loss_workspace_bytes(int64_t B);
int tzk_jrc_loss(const float* logits, int64_t ld, const float* labels, const int64_t* session_ids,
                 const float* weights, int64_t B, float alpha, int32_t key_bits, float* loss, float* dlogits,
                 void* workspace, size_t workspace_bytes, tzk_stream_t stream);

/* ---- RocketLaunching's booster / light head (tzrec/models/rocket_launching.py: the output Linears, the softmax,
 * the softmax cross-entropy of each head, the hint MSE and the feature-based similarity losses), forward and backward.
 * head[0] is the light head, head[1] the booster head (has_booster = 0: light only).  Head e: hidden h [B, H] (rows
 * contiguous), weight w [C, H], bias b [C]; 2 <= C <= 8, 4 <= H <= 1024 with H % 4 == 0.  labels [B] fp32 class
 * indices and losses, or both NULL (no losses: logits and probs only; pairs need labels).  Pair k: light [B, d] and booster [B, d] hidden layers.
 *   head_fwd: logits / probs [B, C] of every head; with labels, losses[3 + n_pairs] =
 *             [0] CE_light, [1] CE_booster, [2] hint = mean (logits_light - logits_booster)^2 over B C,
 *             [3 + k] sim_k: COSINE -0.1 mean_b <normalize(booster), normalize(light)>, EUCLID sqrt(sum (b - l)^2),
 *             CE = the mean over the batch of -sum_c q_c log p_c, q = (1 - eps) onehot(label) + eps / C.
 *             The per-sample terms are summed per CTA and the CTA rows folded in CTA order (partials: grid rows of
 *             3 + n_pairs floats).  pair_stats [n_pairs][B][2] (COSINE) keeps what the backward needs.
 *   head_bwd: dlosses [3 + n_pairs] (device) -> dh of every head, dlight of every pair, dparams = dW_light | db_light
 *             | dW_booster | db_booster as per-CTA partials (grid rows) reduced in CTA order.  No float atomics.
 * The description travels by value as a kernel parameter: graph-capturable. */
#define TZK_ROCKET_MAX_PAIRS 8
#define TZK_ROCKET_MAX_CLASSES 8
#define TZK_ROCKET_COSINE 0
#define TZK_ROCKET_EUCLID 1
typedef struct tzk_rocket_head {
  const float* h;
  const float* w;
  const float* b;
  float* logits;
  float* probs;
  float* dh; /* head_bwd only */
  int32_t H, pad_;
} tzk_rocket_head;
typedef struct tzk_rocket_pair {
  const float* light;
  const float* booster;
  float* dlight; /* head_bwd only */
  int32_t d, pad_;
} tzk_rocket_pair;
typedef struct tzk_rocket_args {
  int64_t B;
  int32_t C, has_booster, n_pairs, sim;
  float eps;
  int32_t pad_;
  const float* labels;
  float* pair_stats;
  tzk_rocket_head head[2];
  tzk_rocket_pair pair[TZK_ROCKET_MAX_PAIRS];
} tzk_rocket_args;
int tzk_rocket_head_fwd(const tzk_rocket_args* args_host, int32_t grid, float* partials, float* losses,
                        tzk_stream_t stream);
int tzk_rocket_head_bwd(const tzk_rocket_args* args_host, const float* dlosses, const float* losses, int32_t grid,
                        float* partials, float* dparams, tzk_stream_t stream);

/* ---- TDM's multi-window DIN attention (tzrec/modules/sequence.py MultiWindowDINEncoder.forward, called from
 * tzrec/models/tdm.py TDM.predict: `self.multiwindow_din(grouped_feature)`), forward and backward over jagged rows.
 * Sample b owns rows offsets[b] .. offsets[b + 1] of seq [N, C] (offsets [B + 1] int64, offsets[0] = 0,
 * offsets[B] = N); query [B, Dq], Dq <= C, zero-padded to C.  Per row at position p < S = sum windows:
 * x = [k, q k, q], h = act(W_l h + b_l) over n_layers attention layers (w[l] [H_l, K_l], K_0 = 3C; act ReLU, or PReLU
 * with one slope per layer), z = lin_w . h + lin_b, a = PReLU(z; act_w).
 *   tdm_fwd: out [B, (L + 1) C] = [window_0 .. window_{L-1}, q], window_w = sum_{p in window w} a_p k_p /
 *            max(min(len - cum_w, W_w), 1); z [N] saved (0 on rows p >= S, which never contribute).
 *   tdm_bwd: d_out [B, (L + 1) C] -> d_seq [N, C], d_query [B, Dq] and dparams = per layer dW [H][K] | db [H] |
 *            dslope [PReLU only], then d lin_w [H_last] | d lin_b | d act_w, as per-CTA partials (grid rows; CTA g owns
 *            samples [B g / grid, B (g + 1) / grid)) reduced in CTA order.  No float atomics.
 * tdm_smem_bytes: the dynamic shared memory of one CTA (backward != 0: of tdm_bwd) for the description's shapes, or
 * 0 outside the cover.  The description travels by value as a kernel parameter: graph-capturable. */
#define TZK_TDM_MAX_LAYERS 3
#define TZK_TDM_MAX_WINDOWS 32
#define TZK_TDM_RELU 0
#define TZK_TDM_PRELU 1
typedef struct tzk_tdm_args {
  int64_t B, N;
  int32_t C, Dq, L, n_layers, act, pad_;
  int32_t windows[TZK_TDM_MAX_WINDOWS];
  int32_t hidden[TZK_TDM_MAX_LAYERS];
  int32_t pad2_;
  const float* seq;
  const int64_t* offsets;
  const float* query;
  const float* w[TZK_TDM_MAX_LAYERS];
  const float* b[TZK_TDM_MAX_LAYERS];
  const float* slope[TZK_TDM_MAX_LAYERS];
  const float* lin_w;
  const float* lin_b;
  const float* act_w;
  float* out;           /* tdm_fwd */
  float* z;             /* written by tdm_fwd, read by tdm_bwd */
  const float* d_out;   /* tdm_bwd only */
  float* d_seq;         /* tdm_bwd only */
  float* d_query;       /* tdm_bwd only */
} tzk_tdm_args;
int64_t tzk_tdm_smem_bytes(const tzk_tdm_args* args_host, int32_t backward);
int tzk_tdm_fwd(const tzk_tdm_args* args_host, int32_t grid, tzk_stream_t stream);
int tzk_tdm_bwd(const tzk_tdm_args* args_host, int32_t grid, float* partials, float* dparams, tzk_stream_t stream);

/* ---- DCN-v2's low-rank cross network (tzrec/modules/interaction.py CrossV2.forward, called from
 * tzrec/models/dcn_v2.py DCNV2.predict: `net = self.cross(net)`), forward and backward.  Per layer l < L:
 *   v_l = U_l x_l (U_l = u_kernels[l].weight [r, D]), w_l = V_l v_l + c_l (V_l = v_kernels[l].weight [D, r],
 *   c_l = v_kernels[l].bias [D]), x_{l+1} = x0 * w_l + x_l;  y = x_L.
 * The tile products run on the tensor cores with the 3xTF32 split (fp32-level results).  Every call first splits the
 * weights it needs into hi / lo TF32 MMA fragments, zero-padded to r8 = r rounded up to 8 and D8 = D rounded up to 8,
 * in `work` (8 L r8 D8 floats, 16-B aligned).
 *   dcn_v2_fwd:         x0 [B, D] -> y [B, D] and the saved v [B, L r].
 *   dcn_v2_bwd_data:    x0, v, dy [B, D] -> dx0 [B, D] and dv [B, L r] (dv_l = d v_l).
 *   dcn_v2_bwd_weight:  x0, v, dv, dy -> dparams = dU [L, r, D] | dV [L, D, r] | dc [L, D], as per-chunk partials
 *                       (`chunks` rows; chunk k owns the k-th of `chunks` equal runs of 64-row batch tiles) reduced in
 *                       chunk order.  No float atomics.
 * dcn_v2_smem_bytes: the dynamic shared memory of one CTA of pass 0 (fwd), 1 (bwd_data) or 2 (bwd_weight) for the
 * description's shapes, or 0 outside the cover (1 <= L <= 8, 1 <= r <= 64, 1 <= D <= 512).  The description travels
 * by value as a kernel parameter: graph-capturable. */
#define TZK_DCN_V2_MAX_LAYERS 8
typedef struct tzk_dcn_v2_args {
  int64_t B;
  int32_t D, L, r, pad_;
  const float* x0;
  const float* wu;      /* [L, r, D] */
  const float* wv;      /* [L, D, r] */
  const float* bias;    /* [L, D] */
  float* work;          /* 8 L r8 D8 floats */
  float* y;             /* dcn_v2_fwd */
  float* v;             /* written by dcn_v2_fwd, read by both backward passes */
  const float* dy;      /* backward */
  float* dx0;           /* dcn_v2_bwd_data */
  float* dv;            /* written by dcn_v2_bwd_data, read by dcn_v2_bwd_weight */
} tzk_dcn_v2_args;
int64_t tzk_dcn_v2_smem_bytes(const tzk_dcn_v2_args* args_host, int32_t pass);
int tzk_dcn_v2_fwd(const tzk_dcn_v2_args* args_host, int32_t grid, tzk_stream_t stream);
int tzk_dcn_v2_bwd_data(const tzk_dcn_v2_args* args_host, int32_t grid, tzk_stream_t stream);
int tzk_dcn_v2_bwd_weight(const tzk_dcn_v2_args* args_host, int32_t chunks, float* partials, float* dparams,
                          tzk_stream_t stream);

/* ---- SelfAttentionEncoder's attention core (tzrec/modules/sequence.py SelfAttentionEncoder.forward: the
 * nn.MultiheadAttention of the in-projected rows, summed over the sequence), forward and backward over jagged rows.
 * Sample b owns rows offsets[b] .. offsets[b + 1] (offsets [B + 1] int64, offsets[0] = 0, offsets[B] = N) of the
 * in-projected q, k, v [N, E] (E = H hd, row strides ldq / ldk / ldv floats); the first L_b = min(len_b, max_len) rows
 * are kept (max_len 0: all).  Per head h over the kept rows: s_ij = (q_i sqrt(1/hd)) . k_j, p = softmax over j.
 *   self_attn_pool_fwd:  pooled [B, E], pooled[b, h] = sum_i sum_j p_ij v_j; lse [N, H] = one log-sum-exp per kept row
 *                        and head (0 on cropped rows).
 *   self_attn_pool_bwd:  d_pooled [B, E] -> dq, dk, dv [N, E] (contiguous; 0 on cropped rows), with the workspace
 *                        dsum [N, H] (D_i = sum_j p_ij u_j, u_j = g . v_j).
 * One CTA per (sample, head) work item at a time, grid-stride: every item writes only its own outputs, so the bits do not
 * depend on the grid.  No float atomics, no host read of any length: graph-capturable.
 * seq_attn_smem_bytes: the dynamic shared memory of one CTA, or 0 outside the cover (1 <= hd <= 128).
 *
 * PoolingEncoder over jagged rows: out [B, D] = sum (mean: / max(L_b, 1)) of the first L_b rows of seq [N, D];
 * jagged_pool_bwd writes d_seq [N, D] = d_out (mean: / max(L_b, 1)) on kept rows and 0 on cropped rows. */
typedef struct tzk_seq_attn_args {
  int64_t B, N;
  int32_t H, hd, max_len, pad_;
  int64_t ldq, ldk, ldv;
  const int64_t* offsets;
  const float* q;
  const float* k;
  const float* v;
  float* pooled;         /* self_attn_pool_fwd */
  float* lse;            /* written by self_attn_pool_fwd, read by self_attn_pool_bwd */
  const float* d_pooled; /* self_attn_pool_bwd only */
  float* dq;             /* self_attn_pool_bwd only */
  float* dk;             /* self_attn_pool_bwd only */
  float* dv;             /* self_attn_pool_bwd only */
  float* dsum;           /* self_attn_pool_bwd workspace [N, H] */
} tzk_seq_attn_args;
int64_t tzk_seq_attn_smem_bytes(const tzk_seq_attn_args* args_host);
int tzk_self_attn_pool_fwd(const tzk_seq_attn_args* args_host, int32_t grid, tzk_stream_t stream);
int tzk_self_attn_pool_bwd(const tzk_seq_attn_args* args_host, int32_t grid, tzk_stream_t stream);
typedef struct tzk_jagged_pool_args {
  int64_t B, N;
  int32_t D, max_len, mean, pad_;
  const int64_t* offsets;
  const float* seq;      /* jagged_pool_fwd */
  float* out;            /* jagged_pool_fwd */
  const float* d_out;    /* jagged_pool_bwd */
  float* d_seq;          /* jagged_pool_bwd */
} tzk_jagged_pool_args;
int tzk_jagged_pool_fwd(const tzk_jagged_pool_args* args_host, int32_t grid, tzk_stream_t stream);
int tzk_jagged_pool_bwd(const tzk_jagged_pool_args* args_host, int32_t grid, tzk_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* TZK_H_ */
