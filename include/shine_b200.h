/*
 * shine_b200.h — C ABI of the H100-native (sm_90a) implementation of SHINE-mapping's per-point SDF
 * training step.  Plain C: raw device pointers + sizes + a cudaStream_t passed as void*; no torch types.
 *
 * The reference (PRBonn/SHINE_mapping @ 0fbaf8a) is 100 % Python and has NO FFI boundary for this path:
 * the path sits behind three Python call sites of the training loop (shine_batch.py:123 `query_feature`,
 * :128 `Decoder.sdf`, :174 `sdf_bce_loss`, :209 `backward`).  Each entry point below names the reference
 * interface it replaces (file:line, relative to the reference root).  INTEGRATION.md shows the ctypes
 * binding a maintainer of the reference would add.
 *
 * Conventions
 *   - return 0 on success, a positive cudaError_t on a CUDA failure, a negative SHINE_ERR_* on a bad
 *     argument / unsupported configuration.  shine_error_string() decodes either.
 *   - all buffers are caller-owned device memory; nothing is allocated, freed or synchronised inside;
 *     every call is asynchronous on `stream` and re-entrant (shine_mesh_export_points, which hands back a count, says
 *     where it waits).  Kernels are launched on the device that owns the
 *     buffers (looked up from the pointers), whatever the calling thread's current device is; a batch on another
 *     device than the tables is SHINE_ERR_INVALID_ARG (pinned host batch pointers are accepted).
 *   - levels are described BOTTOM-UP like `FeatureOctree.hierarchical_indices`
 *     (model/feature_octree.py:201-202): lv[0] is the leaf level `tree_level_world`.
 *   - a voxel that is not in the level's node table is a MISS: its eight corner ids are -1, its feature
 *     contribution is exactly 0 (the reference's zeroed "trash-bin" last row, model/feature_octree.py:76-81,
 *     205-213,232-233) and it receives no gradient.
 */
#ifndef SHINE_B200_H_
#define SHINE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SHINE_ABI_VERSION 5
#define SHINE_MAX_LEVELS 8
#define SHINE_HASH_SLOT_BYTES 64

#define SHINE_OK 0
#define SHINE_ERR_INVALID_ARG (-1)
#define SHINE_ERR_UNSUPPORTED (-2)
#define SHINE_ERR_CAPACITY (-3)   /* an output buffer was too small; what fitted was written */

/* flags of shine_sdf_* calls; each call names the bits it accepts and returns SHINE_ERR_UNSUPPORTED for any other bit
 * (ABI version 3 also defined bit 8) */
#define SHINE_FLAG_REDUCTION_SUM 1u   /* loss_reduction == "sum" (shine_incre.py:77-78); default mean   */
#define SHINE_FLAG_WEIGHTED 2u        /* loss_weight_on (utils/loss.py:18-19): per-sample weight applied */
#define SHINE_FLAG_TF32X1 4u          /* decoder contractions in plain TF32 (default: 3xTF32 ~ fp32)     */
#define SHINE_FLAG_MORTON_ORDERED 16u  /* shine_sdf_step: the batch is in Morton order of its coordinates (the order the
                                         Morton-sorted sample pool hands batches out in).  A hint, never a requirement:
                                         neighbouring points then share nodes, and the step sums the gradients of each run of
                                         equal node on the tensor cores before ONE red per corner row (results equal up to
                                         fp32 summation order); on an unordered batch the flag only costs time           */
#define SHINE_FLAG_LOSS_L2 32u         /* the point-wise loss of shine_sdf_fwd / _step / _eikonal_step: sdf_diff_loss with
                                         l2_loss=True (main_loss_type sdf_l2; shine_batch.py:171-179)                     */
#define SHINE_FLAG_LOSS_L1 64u         /* the same with l2_loss=False (sdf_l1).  Neither loss bit: sdf_bce_loss (sdf_bce);
                                         both: SHINE_ERR_UNSUPPORTED                                                      */

/* One featured level of the FeatureOctree (model/feature_octree.py:46-63). */
typedef struct shine_level {
    const void* hash_slots;   /* capacity x 64-byte slots {u64 morton key | i32 node | pad | i32 ids[8]}:
                                 replaces nodes_lookup_tables[level] (dict morton -> 8 corner rows)      */
    const float* features;    /* hier_features[k]: [rows, F] fp32, last row = trash-bin                  */
    float* feature_grads;     /* same shape, accumulated into (+=); may be NULL when no grads are asked  */
    float* grad_replicas;     /* optional scratch [num_replicas-1, rows, F], all-zero on entry: gradient
                                 privatisation for small (hot) levels — warps spread their red.adds over the
                                 replicas to avoid same-address serialisation in L2; fold them back with
                                 shine_reduce_grad_replicas (which also re-zeroes the scratch)           */
    uint32_t hash_capacity;   /* power of two                                                            */
    int32_t rows;             /* N_l + 1                                                                 */
    int32_t level;            /* octree level in world numbering (leaf = tree_level_world)               */
    int32_t num_replicas;     /* 0/1 = none, else a power of two <= 64                                   */
} shine_level;

typedef struct shine_octree {
    int32_t num_levels;       /* L = tree_level_feat, 1..SHINE_MAX_LEVELS                                */
    int32_t feature_dim;      /* F = feature_dim (multiple of 4; fused sdf_* kernels need 8)             */
    int32_t poly_interp;      /* poly_int_on: smoothstep 3d^2-2d^3 weights (model/feature_octree.py:176) */
    int32_t reserved;
    shine_level lv[SHINE_MAX_LEVELS];
} shine_octree;

/* Geometry decoder (model/decoder.py:29-36): Linear(F,H)+ReLU, Linear(H,H)+ReLU, Linear(H,1);
 * PyTorch (out,in) row-major weights.  Bias pointers may be NULL (geo_mlp_bias_on False).
 * g* are gradient buffers (+=); all NULL == frozen decoder (utils/tools.py:188-191). */
typedef struct shine_decoder {
    const float *w1, *b1, *w2, *b2, *w3, *b3;
    float *gw1, *gb1, *gw2, *gb2, *gw3, *gb3;
    int32_t in_dim;           /* F  (8)  */
    int32_t hidden;           /* H  (32) */
    int32_t mlp_level;        /* 2       */
    int32_t reserved;
} shine_decoder;

int shine_abi_version(void);
const char* shine_error_string(int code);

/* Build / extend the device node table of one level.  Replaces the Python dict fill at
 * model/feature_octree.py:162-166.  `slots` must have been memset to 0xFF (empty) before the first
 * insert.  keys: [n] int64 Morton codes, corner_ids: [n,8] int32 rows, node_base: ordinal of keys[0].
 * overflow_count (device int32, may be NULL): incremented once per key that could NOT be stored because the
 * table is full — a Python dict never drops a key, so the caller must grow the table and re-insert. */
int shine_hash_insert(void* slots, uint32_t capacity, const int64_t* keys, const int32_t* corner_ids,
                      int64_t n, int32_t node_base, int32_t* overflow_count, void* stream);

/* kal.ops.spc.quantize_points + points_to_morton (call sites model/feature_octree.py:203-204):
 * coord [n,3] fp32 -> morton [n] int64 at `level`. */
int shine_points_to_morton(const float* coord, int64_t n, int32_t level, int64_t* morton, void* stream);

/* FeatureOctree.get_indices (model/feature_octree.py:199-218): out_idx [L, n, 8] int64, level-major
 * bottom-up, -1 x8 on a miss. */
int shine_get_indices(const shine_octree* oct, const float* coord, int64_t n, int64_t* out_idx, void* stream);

/* FeatureOctree.query_feature (model/feature_octree.py:237-244; interpolat :172-196, blend :222-234):
 * out_feat [n, F] fp32 = sum over levels of the 8-corner blend. */
int shine_query_fwd(const shine_octree* oct, const float* coord, int64_t n, float* out_feat, void* stream);

/* autograd of the above (the index_put_(accumulate=True) of shine_batch.py:209):
 * lv[i].feature_grads[id] += w_c * dfeat[p]  for every hit corner. */
int shine_query_bwd(const shine_octree* oct, const float* coord, int64_t n, const float* dfeat, void* stream);

/* Coordinate derivatives of query_feature, for the eikonal / normal terms that the reference obtains with
 * torch.autograd.grad(pred, coord, create_graph=True) (utils/tools.py:175-185, shine_batch.py:141-142,183-185).
 * With dw_c/da the derivative of the interpolation weight of corner c w.r.t. axis a (incl. the smoothstep and the
 * 2^level/2 scaling of model/feature_octree.py:173-178):
 *   coord_grad : out_dcoord[p][a]  = sum_levels sum_c dw_c/da * <features[id_c], dfeat[p]>            ([n,3])
 *   tangent_fwd: out[p][:]         = sum_levels sum_c (sum_a tangent[p][a] dw_c/da) * features[id_c]   ([n,F])
 *   tangent_bwd: feature_grads[id_c] += (sum_a tangent[p][a] dw_c/da) * dfeat[p]
 * coord_grad is the backward of query_fwd w.r.t. coord; tangent_fwd / tangent_bwd are coord_grad's own backward
 * w.r.t. dfeat / the tables (double backward). */
int shine_query_coord_grad(const shine_octree* oct, const float* coord, int64_t n, const float* dfeat,
                           float* out_dcoord, void* stream);
int shine_query_tangent_fwd(const shine_octree* oct, const float* coord, int64_t n, const float* tangent,
                            float* out_feat, void* stream);
int shine_query_tangent_bwd(const shine_octree* oct, const float* coord, int64_t n, const float* tangent,
                            const float* dfeat, void* stream);

/* query_feature -> Decoder.sdf (model/decoder.py:49-63) fused, forward only (the mesher's query,
 * utils/mesher.py:60-72).  out_pred [n].  out_mask (optional, may be NULL) [n] uint8 = voxel present at
 * lv[mask_level] (utils/mesher.py:82-89). */
int shine_sdf_infer(const shine_octree* oct, const shine_decoder* dec, const float* coord, int64_t n,
                    float* out_pred, uint8_t* out_mask, int32_t mask_level, uint32_t flags, void* stream);

/* query_feature -> Decoder.sdf -> the point-wise loss (shine_batch.py:171-179), forward only.  The loss bits of flags
 * pick the loss; with z = sigmoid(label / sigma) and d = (pred - label) / scale (metres):
 *   sdf_bce (no loss bit)   sdf_bce_loss  (utils/loss.py:17-24)  L = sum w (max(pred, 0) - pred z + log(1 + exp(-|pred|)))
 *                           with w = |weight| under SHINE_FLAG_WEIGHTED, else 1
 *   sdf_l1 (LOSS_L1)        sdf_diff_loss (utils/loss.py:6-14)   L = sum |weight| |d|
 *   sdf_l2 (LOSS_L2)        sdf_diff_loss, l2_loss=True          L = sum |weight| d^2
 * label [n]; weight [n], or NULL for sdf_bce without SHINE_FLAG_WEIGHTED; sigma = sigma_sigmoid (shine_batch.py:87),
 * > 0 for sdf_bce; scale = config.scale (1 / world_size), positive and finite for sdf_l1 / sdf_l2.  Each loss ignores the
 * other's parameter.  out_loss [1] fp32 is ACCUMULATED (+=): caller zeroes it.  loss_scale multiplies every per-point
 * term: 1/N_global for "mean" and for sdf_l1 / sdf_l2 (the reference's count), 1 for "sum".
 * flags: sdf_bce SHINE_FLAG_REDUCTION_SUM | WEIGHTED | TF32X1 | MORTON_ORDERED (the reduction is loss_scale's, the order
 * a hint of the step's); sdf_l1 / sdf_l2 only SHINE_FLAG_TF32X1 besides the loss bit (sdf_diff_loss always weighs by
 * |weight| and divides by the count).  Any other bit is SHINE_ERR_UNSUPPORTED, checked first. */
int shine_sdf_fwd(const shine_octree* oct, const shine_decoder* dec, const float* coord, const float* label,
                  const float* weight, int64_t n, float sigma, float scale, float loss_scale, float* out_pred,
                  float* out_loss, uint32_t flags, void* stream);

/* The whole training step shine_batch.py:123-209 in ONE pass: forward, loss (as shine_sdf_fwd) and the backward that
 * scatter-adds into lv[i].feature_grads and dec->g*.  d_loss: device scalar dL/dloss (NULL == 1).
 * out_pred / out_loss may be NULL (pure backward == "recompute" mode for a separate autograd backward).  flags as
 * shine_sdf_fwd, and SHINE_FLAG_MORTON_ORDERED with sdf_l1 / sdf_l2 too. */
int shine_sdf_step(const shine_octree* oct, const shine_decoder* dec, const float* coord, const float* label,
                   const float* weight, int64_t n, float sigma, float scale, float loss_scale, const float* d_loss,
                   float* out_pred, float* out_loss, uint32_t flags, void* stream);

/* shine_sdf_fwd with sdf_bce_loss (either loss bit is SHINE_ERR_UNSUPPORTED), under the name and arguments of ABI
 * version 4, which benchmark scripts bind. */
int shine_sdf_bce_fwd(const shine_octree* oct, const shine_decoder* dec, const float* coord,
                      const float* label, const float* weight, int64_t n, float sigma, float loss_scale,
                      float* out_pred, float* out_loss, uint32_t flags, void* stream);

/* feature_grads[l] += sum of grad_replicas[l][r]; grad_replicas[l] = 0.  No-op for levels without
 * replicas.  Part of the backward (the reference's index_put_ is one pass, shine_batch.py:209). */
int shine_reduce_grad_replicas(const shine_octree* oct, void* stream);

/* Dense Adam (utils/tools.py:78-79: betas (0.9,0.99), eps 1e-15, weight decay as L2 on grads) over up to
 * SHINE_ADAM_MAX_TENSORS tensors in one launch — shine_batch.py:210 `opt.step()`. */
#define SHINE_ADAM_MAX_TENSORS 16
typedef struct shine_adam_tensor {
    float* param; float* grad; float* exp_avg; float* exp_avg_sq;
    int64_t numel; float lr; float weight_decay;
} shine_adam_tensor;
int shine_adam_step(const shine_adam_tensor* tensors, int32_t count, float beta1, float beta2, float eps,
                    int32_t step, int32_t zero_grad, void* stream);

/* Same, CUDA-graph friendly: the step number lives on the device.  state = {int32 step, f32 bc1, f32 bc2_sqrt}
 * (12 bytes, zero-initialised by the caller once); every call increments step and refreshes the bias
 * corrections in a 1-thread kernel, then runs the Adam kernel reading them — so a captured graph can be replayed. */
int shine_adam_step_dev(const shine_adam_tensor* tensors, int32_t count, float beta1, float beta2, float eps,
                        void* state, int32_t zero_grad, void* stream);

/* ---- FeatureOctree.update on the GPU (model/feature_octree.py:114-166) ---------------------------------------------
 * All featured levels of one scan at once; lv[] here is coarse -> fine; world levels 1 .. 15 (kaolin's int16 points).
 * Scratch (frame-local key sets, lists) is caller-owned; sets are arrays of u64 filled with 0xFF, capacity a power of
 * two >= 2x the insertions.
 * Sequence: frame_nodes -> (host reads new_node_count, sizes tables, copies the N node entries to the front of the sort
 * input and points new_corner_keys right behind them) -> frame_corners -> (host reads new_corner_count) ->
 * sort_new_keys over the N + C entries -> assign_rows (the first C sorted entries) -> fill_nodes (the last N).
 * Row numbering is the reference's: unseen corners of the new nodes, unique, in lexicographic (x, y, z) order of
 * kaolin's int16 points, appended after the existing rows (:131-151).  Node numbering too: new nodes in ascending
 * Morton order, appended (:164-166). */
typedef struct shine_build_level {
    void* node_slots;               /* the level's node table (64-byte slots), NULL while the level is empty          */
    void* corner_slots;             /* the level's corner table: 16-byte slots {u64 lexicographic key, i32 row, pad} */
    void* frame_node_set;           /* scratch u64 set                                                                */
    void* frame_corner_set;         /* scratch u64 set (frame_corners onwards)                                        */
    int32_t* node_ids_out;          /* out [new nodes, 8] corner rows of those nodes, Morton order (fill_nodes)       */
    int64_t* corner_morton_out;     /* out [new corners] Morton code of each new row, in row order (assign_rows)      */
    uint32_t node_capacity, corner_capacity, frame_node_set_capacity, frame_corner_set_capacity;
    int32_t level;                  /* world level                                                                    */
    int32_t nodes_before, rows_before;   /* nodes / corner rows (without the trash row) the level already holds       */
    int32_t reserved;
} shine_build_level;
typedef struct shine_build {
    int32_t num_levels, max_level;
    int32_t* new_node_count;        /* device [L], zero on entry                                                      */
    int32_t* new_corner_count;      /* device [L], zero on entry                                                      */
    int32_t* new_corner_total;      /* device [1], zero on entry                                                      */
    int32_t* new_node_total;        /* device [1], zero on entry                                                      */
    uint64_t* new_node_keys;        /* out [<= L * n points] (1 << 51) | (level index << 45) | Morton key, unordered  */
    uint64_t* new_corner_keys;      /* scratch [8 * sum new nodes]: (level index << 48) | lexicographic key           */
    shine_build_level lv[SHINE_MAX_LEVELS];
} shine_build;

int shine_octree_frame_nodes(const shine_build* plan, const float* points, int64_t n, void* stream);
int shine_octree_frame_corners(const shine_build* plan, int32_t new_nodes, void* stream);
int64_t shine_octree_sort_scratch_bytes(int32_t n);
int shine_octree_sort_new_keys(const void* keys_in, void* keys_out, int32_t n, void* scratch, int64_t scratch_bytes,
                               void* stream);
int shine_octree_assign_rows(const shine_build* plan, const void* sorted_keys, int32_t total, void* stream);
/* sorted_nodes: the last new_nodes entries of the sort output; their tags are cleared in place (plain Morton keys) */
int shine_octree_fill_nodes(const shine_build* plan, void* sorted_nodes, int32_t new_nodes, int32_t* overflow_count,
                            void* stream);
/* rebuild a corner table from the per-row Morton codes (after growing it, moving devices or unpickling) */
int shine_octree_corner_rehash(void* corner_slots, uint32_t capacity, const int64_t* corner_morton_by_row, int64_t rows,
                               void* stream);

/* ---- the step with `ekional_loss_on` (config/kitti/kitti_batch.yaml:46) as one kernel ---------------------------------
 * Replaces shine_batch.py:119-142,172-185,208-209 + utils/tools.py:175-185 (autograd.grad(pred, coord, create_graph=True)
 * and the double backward through gather, decoder and loss):
 *   g = sigma * d pred / d coord;   L = point-wise loss(pred, label) + weight_e * mean_{weight > 0} (1 - |g|)^2
 * The point-wise loss is shine_sdf_fwd's, picked by the same loss bits; sigma = sigma_sigmoid, > 0 whatever the loss.
 * Accumulates dL/d(tables) into lv[i].feature_grads and dL/d(decoder) into dec->g* (both terms).
 *   weight     [n]: sign marks surface (+) / free-space (-) samples (shine_batch.py:137); |weight| multiplies the sdf_bce
 *              term only with SHINE_FLAG_WEIGHTED, the sdf_l1 / sdf_l2 term always
 *   n_surface  device int32: number of samples with weight > 0 (shine_count_positive) in the whole batch; when this call
 *              sees one part of it (a rank's shard, a chunk), the count of the whole batch; 0 -> no eikonal contribution
 *   out_pred [n] / out_grad [n,3] (g) may be NULL; out_loss (+=) the point-wise part; out_eikonal (+=) the mean, without
 *              weight_e
 * flags: sdf_bce SHINE_FLAG_REDUCTION_SUM | WEIGHTED | TF32X1 (the reduction is loss_scale's); sdf_l1 / sdf_l2 only
 * SHINE_FLAG_TF32X1 besides the loss bit.  TF32X1 is accepted and changes nothing: the kernel is fp32 throughout.  Any
 * other bit is SHINE_ERR_UNSUPPORTED. */
int shine_count_positive(const float* values, int64_t n, int32_t* out_count, void* stream);
int shine_sdf_eikonal_step(const shine_octree* oct, const shine_decoder* dec, const float* coord, const float* label,
                           const float* weight, int64_t n, float sigma, float scale, float loss_scale, float weight_e,
                           const int32_t* n_surface, float* out_pred, float* out_grad, float* out_loss,
                           float* out_eikonal, uint32_t flags, void* stream);

/* ---- continual-learning terms of the incremental loop (BASELINE config 4) ---------------------------------------
 * The reference finds the rows a batch touched with `hierarchical_indices[i].flatten().unique()` (a sort per level
 * per step, model/feature_octree.py:251) and then works on dense [rows, F] tensors.  Here the touched rows of a batch
 * are a compact per-level list: one bit per row in `bitmap` (all zero between uses), first setter appends the row. */
typedef struct shine_touched_level {
    uint32_t* bitmap;         /* [(rows + 31) / 32] words, zero on entry                                       */
    int32_t* rows;            /* [capacity] touched row ids, unordered, each row once                           */
    int32_t* count;           /* device scalar, zero on entry                                                   */
    int32_t capacity;         /* >= min(rows, 8 n)                                                              */
    int32_t reserved;
} shine_touched_level;
typedef struct shine_touched { shine_touched_level lv[SHINE_MAX_LEVELS]; } shine_touched;   /* bottom-up like shine_octree */

/* per-level row-aligned side tables of the incremental loop, bottom-up: features_last_frame / importance_weight
 * (model/feature_octree.py:70-72) */
typedef struct shine_row_tables {
    const float* last[SHINE_MAX_LEVELS];        /* features_last_frame (regularisation)                       */
    const float* importance[SHINE_MAX_LEVELS];  /* importance_weight, read  (regularisation)                  */
    float* importance_rw[SHINE_MAX_LEVELS];     /* importance_weight, updated (importance pass)               */
} shine_row_tables;

/* Collect the rows touched by `coord` (hit voxels only: the reference's -1 row has zero importance,
 * utils/incre_learning.py:40).  Replaces the unique() of model/feature_octree.py:251. */
int shine_mark_touched(const shine_octree* oct, const float* coord, int64_t n, const shine_touched* touched,
                       void* stream);

/* FeatureOctree.cal_regularization (model/feature_octree.py:246-255) and its gradient, over the touched rows only:
 *   *out_reg (+=)         sum_u Omega[u] * (f[u] - f_last[u])^2
 *   feature_grads[u] +=   grad_scale * Omega[u] * (f[u] - f_last[u])        (grad_scale = 2 * lambda_forget)
 * clear_marks != 0 also clears the bitmap bits of the processed rows (leave it 0 when another pass follows). */
int shine_regularization_apply(const shine_octree* oct, const shine_touched* touched, const shine_row_tables* aux,
                               float grad_scale, float* out_reg, int32_t clear_marks, void* stream);

/* cal_feature_importance's accumulation (utils/incre_learning.py:36-40) over the touched rows only:
 *   importance_rw[u] += |feature_grads[u]|;  zero_grads != 0: feature_grads[u] = 0 afterwards (:38). */
int shine_importance_accumulate(const shine_octree* oct, const shine_touched* touched, const shine_row_tables* aux,
                                int32_t zero_grads, int32_t clear_marks, void* stream);

/* ---- the sample pool of incremental mapping with replay (continual.window_replay_on) -------------------------------
 * Structure of arrays, fp32, device memory of one GPU; samples [0, size) are the pool, [size, capacity) free room. */
typedef struct shine_sample_pool {
    float* coord; float* label; float* weight;   /* [capacity,3], [capacity], [capacity] fp32, device                  */
    int64_t size, capacity;
} shine_sample_pool;

/* Bytes of caller scratch that shine_pool_window_append needs for size + n_new samples (tile counter and one status word
 * per 2048-sample tile); SHINE_ERR_INVALID_ARG for a negative count. */
int64_t shine_pool_scratch_bytes(int64_t n_total);

/* Replaces dataset/lidar_dataset.py:237-251 (drop the pool samples at `window_radius * scale` or more from the new frame's
 * origin: `(coord_pool - origin).norm(2, dim=-1) < r` and the masked gathers of coord, weight and sdf_label) followed by
 * :263-270 (`torch.cat` of the frame's samples), as ONE launch, in place, in the reference's order:
 *   pool = [old samples with sqrt((dx*dx + dy*dy) + dz*dz) < radius, fp32 without contraction | the n_new frame samples]
 * radius is the fp32 value the reference compares with (float32(window_radius * scale), the product taken in double);
 * the comparison is strict and a NaN coordinate is dropped.  The new size goes to the device int64 *size_out.
 * pool->size + n_new must not exceed pool->capacity.  The frame buffers (coord [n_new,3], label, weight) must not overlap
 * the pool; they are device memory of the pool's GPU or pinned host memory.  scratch: >= shine_pool_scratch_bytes of
 * size + n_new, 8-byte aligned, device memory of the pool's GPU; cleared on `stream` by this call. */
int shine_pool_window_append(const shine_sample_pool* pool, const float* coord, const float* label, const float* weight,
                             int64_t n_new, float ox, float oy, float oz, float radius, int64_t* size_out, void* scratch,
                             int64_t scratch_bytes, void* stream);

/* ---- one LiDAR frame from its file's records to training samples ---------------------------------------------------
 * Replaces dataset/lidar_dataset.py:115-218 (process_frame: preprocess_kitti :334-339, open3d crop :139-142, voxel
 * down-sampling :158, transform :179 and scale :189) and utils/data_sampler.py:18-139 (dataSampler.sample).
 * Records are the file's bytes as read: n records of stride_bytes, x y z first, float32 (fp64 = 0) or float64 (fp64 = 1).
 * The four calls run in order on one scratch (>= shine_scan_scratch_bytes(n), 256-byte aligned, device memory) and the
 * same records; only the voxel count has to reach the host between the second and the third. */
typedef struct shine_scan_input {
    const void* records;    /* device [n * stride_bytes] */
    int64_t n;
    int32_t stride_bytes;
    int32_t fp64;
} shine_scan_input;

int64_t shine_scan_scratch_bytes(int64_t n);
/* Keeps, in fp64, z > min_z, sqrt((x*x + y*y) + z*z) >= min_range and -r <= x, y <= r, min_z <= z <= max_z (NaN and inf
 * points fail); takes the per-axis bounds of the kept points and their voxel keys floor((p - (min - v/2)) / v), 21 bits
 * per axis.  A crop box wider than 2^21 - 2 voxels on an axis is SHINE_ERR_INVALID_ARG. */
int shine_scan_filter_keys(const shine_scan_input* in, double min_z, double max_z, double min_range, double pc_radius,
                           double voxel, void* scratch, int64_t scratch_bytes, void* stream);
/* Stable radix sort of (key, input index); the number of voxels goes to the device int64 *voxel_count. */
int shine_scan_sort_voxels(int64_t n, int64_t* voxel_count, void* scratch, int64_t scratch_bytes, void* stream);
/* Voxel i (ascending key) = fp64 sum of its points in input order / their count -> voxels_out[i] (nullable, [n_voxels,3]
 * fp64); then q = pose·[p,1] (row-major 4x4, host memory; rows ((m0*x + m1*y) + m2*z) + m3, no FMA), q.xyz / q.w, times
 * scale, rounded to nearest fp32 -> points_out [n_voxels,3]. */
int shine_scan_average_transform(const shine_scan_input* in, const double* pose, double scale, int64_t n_voxels,
                                 double* voxels_out, float* points_out, void* scratch, int64_t scratch_bytes,
                                 void* stream);
/* dataSampler.sample in fp32 without contraction, for n_rays points and the sensor origin (ox, oy, oz).  Uniforms are
 * sample-major like the reference's torch.rand(R*n, 1): u_surface[s*R + i] is surface sample s of ray i.
 * Per ray i, output rows i*(surface_n + free_n) + s: surface samples then free-space samples; coord = shift*ratio + o,
 * label = displacement, weight = +1 (surface) / -1 (free).  surface_range, free_end: the fp32 values of
 * surface_sample_range_m * scale and free_sample_end_dist_m * scale. */
int shine_scan_sample(const float* points, int64_t n_rays, float ox, float oy, float oz, const float* u_surface,
                      int32_t surface_n, const float* u_free, int32_t free_n, float surface_range, float free_end,
                      float free_begin_ratio, float* coord, float* label, float* weight, void* stream);

/* ---- one depth image to camera points (dataset/rgbd_to_kitti_format.py: open3d's create_from_color_and_depth and
 * create_from_rgbd_image) ------------------------------------------------------------------------------------------
 * Pixel (i, j), i < height, j < width, is depth[i * row_pitch + j] (device uint16, 2-byte aligned).  d = (float)raw /
 * (float)depth_scale in fp32, set to 0 when (double)d >= depth_trunc.  A pixel with d > 0 gives, in fp64 with every
 * operation rounded on its own, z = d, x = ((j - cx) * z) / fx, y = ((i - cy) * z) / fy and
 * xyz_out[i * width + j] = rows 0..2 of camera_pose · (x, y, z, 1) (row-major 4x4, host memory; each row
 * ((m0 x + m1 y) + m2 z) + m3 · 1; row 3 is not read); every other pixel gives (NaN, NaN, NaN).  xyz_out: device
 * [height * width, 3] fp64, 8-byte aligned, row-major pixel order, which shine_scan_* take as 24-byte fp64 records (their
 * filter drops the NaN records).  rgb_out / rgb_in: both NULL, or device uint8 rgb_out[i * width + j] = rgb_in[i *
 * row_pitch + j] (3 bytes each) for every pixel.  NULL pointers, height or width < 1, row_pitch < width and depth_scale
 * <= 0 (or not a positive finite fp32) are SHINE_ERR_INVALID_ARG, height * row_pitch > 2^31 - 1 is
 * SHINE_ERR_UNSUPPORTED; none of them launches.  One launch, no allocation, no synchronisation. */
int shine_rgbd_backproject(const uint16_t* depth, int32_t height, int32_t width, int32_t row_pitch, double fx,
                           double fy, double cx, double cy, double depth_scale, double depth_trunc,
                           const double* camera_pose, double* xyz_out, uint8_t* rgb_out, const uint8_t* rgb_in,
                           void* stream);

/* ---- the batch-mode sample pool in pinned host memory (more than `pc_count_gpu_limit` scans) ------------------------
 * Replaces the CPU pools of dataset/lidar_dataset.py:94-101 and the CPU-side gather + copy of get_batch (:431-448).
 * Record i is 32 bytes, 32-byte aligned, {x, y, z, label, weight, 0, 0, 0} fp32, at byte (i & (2^chunk_shift - 1)) * 32 of
 * chunk i >> chunk_shift.  Chunks are pinned (page-locked) host memory the GPU addresses directly (unified addressing);
 * `chunks` is a DEVICE array of num_chunks such pointers, on the GPU that runs the kernels. */
typedef struct shine_host_pool {
    void* const* chunks;      /* device [num_chunks] pointers to pinned host chunks of 2^chunk_shift records each        */
    int32_t chunk_shift;      /* 5 .. 31                                                                                  */
    int32_t num_chunks;
    int64_t size;             /* records in the pool: gather indices must lie in [0, size); <= num_chunks << chunk_shift   */
} shine_host_pool;

/* Pack a frame's device samples (coord [n,3], label [n], weight [n] fp32) into records at + 0 .. at + n - 1 (one launch;
 * the run may cross chunk boundaries).  at + n must not exceed num_chunks << chunk_shift; `size` is not read or changed. */
int shine_host_pool_append(const shine_host_pool* pool, int64_t at, const float* coord, const float* label,
                           const float* weight, int64_t n, void* stream);

/* The batch of get_batch: coord_out[t] = (x, y, z), label_out[t], weight_out[t] of record index[t], t < n (int64 device
 * indices; device outputs [n,3], [n], [n]).  One launch, no host synchronisation: capturable in a CUDA graph.  An index
 * outside [0, size) gives NaN coordinates and label = weight = 0. */
int shine_host_pool_gather(const shine_host_pool* pool, const int64_t* index, int64_t n, float* coord_out,
                           float* label_out, float* weight_out, void* stream);

/* ---- multi-GPU exchange (SURVEY.md 8e, 8b export (6); the reference is single-GPU) --------------------------------
 * One process per GPU.  The map is partitioned by Morton prefix at the coarsest featured level; every rank owns the
 * rows reachable from its blocks, so corner rows on a face between two blocks exist on both ranks.  Their gradients
 * are summed through a compact exchange buffer laid out [decoder grads | boundary rows of lv[0] | lv[1] | ...]:
 * pack -> ONE all-reduce (decoder + boundary) -> unpack. */
typedef struct shine_boundary_level {
    float* table;             /* this rank's [rows, F] gradient (or feature) table of the level                 */
    const int32_t* rows;      /* [count] local rows that are shared with another rank                           */
    const int32_t* slots;     /* [count] their positions in the level's globally agreed boundary list           */
    int64_t offset;           /* float offset of the level's segment in the exchange buffer (multiple of 4)     */
    int32_t count;
    int32_t reserved;
} shine_boundary_level;
typedef struct shine_boundary { shine_boundary_level lv[SHINE_MAX_LEVELS]; } shine_boundary;

/* buf[offset_l + slot * F ..] = table_l[row]   /   table_l[row] = buf[offset_l + slot * F ..] */
int shine_boundary_pack(const shine_boundary* plan, int32_t num_levels, int32_t feature_dim, float* buf, void* stream);
int shine_boundary_unpack(const shine_boundary* plan, int32_t num_levels, int32_t feature_dim, float* buf, void* stream);

/* NCCL communicator owned by this library (NCCL is bound with dlopen at run time).  Rank 0 makes the 128-byte
 * unique id, the caller distributes it (any transport), every rank creates its communicator on `device`. */
int shine_nccl_unique_id(void* out_id128);
int shine_nccl_comm_create(const void* id128, int32_t nranks, int32_t rank, int32_t device, void** out_comm);
int shine_nccl_comm_destroy(void* comm);
/* In-place sum all-reduce of `count` floats over NVLink, asynchronous on `stream`: the decoder-gradient exchange
 * that follows the backward (comm is the ncclComm_t made above, or any ncclComm_t of the same NCCL).
 * NCCL failures return -1000 - ncclResult_t; shine_comm_last_error() has the text. */
int shine_allreduce_decoder_grads(void* comm, float* buf, int64_t count, void* stream);
const char* shine_comm_last_error(void);

/* The same exchange as ONE kernel over NVLink peer memory (no NCCL): pack own [decoder | boundary rows] into an
 * IPC-shared buffer, publish a step flag into every peer's buffer, wait for the peers' flags, sum all ranks' buffers
 * in fixed rank order straight over NVLink, in place into dec_grads / the plan's table rows.  One process per GPU:
 * create (returns the 64-byte cudaIpcMemHandle_t of this rank's buffer) -> the caller all-gathers the handles ->
 * connect -> exchange every step (all ranks, same order).  plan offsets are relative to the exchange buffer whose first
 * dec_floats floats are the decoder segment, exactly as for shine_boundary_pack.  A peer that never shows up is a
 * counted timeout (shine_p2p_timeouts), not a hang. */
typedef struct shine_boundary_inverse {
    const int32_t* row_of_slot[SHINE_MAX_LEVELS];   /* [slots of the level] local row holding that shared corner, -1 if none */
    int32_t slots[SHINE_MAX_LEVELS];                /* length of the level's globally agreed boundary list           */
    const int32_t* holders[SHINE_MAX_LEVELS];       /* [slots] bit r set: rank r holds a row of that corner (its buffer is
                                                       read for the sum); NULL: every rank's buffer is read            */
} shine_boundary_inverse;
typedef struct shine_p2p shine_p2p;
int shine_p2p_create(int32_t nranks, int32_t rank, int32_t device, int64_t max_floats, void* out_handle64, shine_p2p** out);
int shine_p2p_connect(shine_p2p* ctx, const void* handles /* nranks x 64 B, rank order */);
int shine_p2p_exchange(shine_p2p* ctx, float* dec_grads, int64_t dec_floats, const shine_boundary* plan,
                       const shine_boundary_inverse* inverse, int32_t num_levels, int32_t feature_dim, void* stream);
int shine_p2p_timeouts(shine_p2p* ctx, int32_t* out_count);
int shine_p2p_destroy(shine_p2p* ctx);

/* ---- meshing: utils/mesher.py recon_octree_mesh / recon_bbx_mesh -------------------------------------------------
 * The grid of the marching cubes is block-sparse: bricks of n^3 cubes at integer brick coordinates B; brick B owns the
 * grid indices G = B n + (i, j, k), 0 <= i, j, k < n, and stores them together with its +1 faces ((n+1)^3 points, the
 * corners of all its cubes), so that one chunk of bricks can be queried and meshed without the others.  Grid index G
 * is the point origin + spacing * G (fp32: __fadd_rn(origin, __fmul_rn(spacing, G))) of the [-1,1] cube.  Grid
 * indices must lie in [0, 2^20). */
typedef struct shine_brick_grid {
    const int32_t* bricks;    /* [num_bricks, 3] brick coordinates of this chunk                                        */
    float* sdf;               /* [num_bricks, (n+1)^3] fp32, point (i,j,k) at (i (n+1) + j) (n+1) + k                   */
    uint8_t* mask;            /* same layout                                                                             */
    const int64_t* all_keys;  /* ascending keys (Bx << 42) | (By << 21) | Bz of every brick of the map, or NULL          */
    int64_t num_all;
    int64_t num_bricks;
    float origin[3];
    float spacing;
    int32_t n;                /* cubes per brick side, 1 .. 64                                                           */
    int32_t lo[3];            /* vertices are written relative to grid index lo                                         */
    int32_t hi[3];            /* the cube at lowest corner G is processed iff mask[G] and G + 1 < hi on every axis        */
    float missing_sdf;        /* value of a +1 face point whose brick is not in all_keys (its mask is 0)                */
} shine_brick_grid;

/* Fills sdf = -Decoder.sdf(query_feature(p)) and mask = voxel present at lv[mask_level] (utils/mesher.py:60-89) at every
 * point of the chunk, with the same kernel as shine_sdf_infer (flags as there).  With all_keys, +1 face points of bricks
 * missing from all_keys then get missing_sdf and mask 0 (the zero-initialised global grid of utils/mesher.py:323-324). */
int shine_mesh_grid(const shine_octree* oct, const shine_decoder* dec, const shine_brick_grid* grid, int32_t mask_level,
                    uint32_t flags, void* stream);

/* Masked marching cubes (skimage.measure.marching_cubes(sdf, 0, mask=mask, allow_degenerate=False), as used by
 * utils/mesher.py:216-217) over one chunk of a shine_mesh_grid-filled grid, in two calls per chunk:
 *   count (verts == NULL): every sign-changing edge (one corner < 0, the other >= 0) of a processed cube is entered in the
 *     edge table (16-byte slots, memset to 0xFF before the first chunk, kept across the chunks of one mesh) and new
 *     edges are numbered from counters[0]; counters[1] += the chunk's triangles without two coincident vertices;
 *     counters[3] counts edges that did not fit (the caller must start over with a larger table).
 *   emit (verts != NULL, after the host read counters[0..1]): verts[id] = position of the edge's vertex, t = v0 / (v0 - v1)
 *     along the edge, in grid units relative to lo (fp32 [vert_capacity, 3]); the chunk's triangles (int32 vertex ids,
 *     [tri_capacity, 3]) go to rows counters[2] onwards, counters[2] advancing. */
int shine_marching_cubes(const shine_brick_grid* grid, void* edge_slots, uint32_t edge_capacity, int32_t* counters,
                         float* verts, int64_t vert_capacity, int32_t* tris, int64_t tri_capacity, void* stream);

/* save_map (utils/mesher.py:152-173 generate_sdf_map): the grid points of one shine_mesh_grid-filled chunk as the body of a
 * binary little-endian PLY, 20-byte records {float x, y, z, intensities; int32 labels}.  Only the points a brick OWNS are
 * written (i, j, k < n: its +1 face points belong to a neighbour or are padding, so no point is written twice), and of
 * those the ones with G < hi on every axis and, with masked_only, mask != 0.
 *   position    = transform (3x4 fp64, row-major, host) applied to origin_m + voxel_m (G - lo) (fp64, host; origin_m is
 *                 the position of grid index lo in metres): ((t0 x + t1 y) + t2 z) + t3 per row, every operation rounded
 *                 on its own, then rounded to fp32;
 *   intensities = sdf * sdf_factor in fp32 (the buffer holds -Decoder.sdf, the sign of the reference's sdf_pred; with
 *                 sdf_factor = logistic_gaussian_ratio * sigma_sigmoid_m this is metres, positive in free space);
 *   labels      = mask != 0.
 * Record r of the call goes to records[20 (c + r)], c = *counter on entry (device int64, zeroed by the caller before the
 * first chunk of a buffer); the order of the records is unspecified.  Records at index >= capacity are counted, not
 * written.  Unlike the other entry points this one WAITS for its kernel: it returns with *count_out (host, optional) =
 * *counter, and SHINE_ERR_CAPACITY when that exceeds capacity.  records (4-byte aligned), counter and the grid's buffers
 * must be on one device. */
int shine_mesh_export_points(const shine_brick_grid* grid, const double* origin_m, double voxel_m, const double* transform,
                             float sdf_factor, int32_t masked_only, void* records, int64_t capacity, int64_t* counter,
                             int64_t* count_out, void* stream);

/* Open3D's compute_vertex_normals and cluster_connected_triangles as used by utils/mesher.py:240-249,278-281:
 * normals [nv, 3] = normalised sum of the unit normals of the adjacent triangles; keep[t] = 1 iff the cluster of
 * triangles connected through shared edges that holds t has at least min_tris triangles.  edge_slots: 16-byte slots,
 * capacity a power of two >= 2 * 3 nt, memset to 0xFF; scratch: int32 [2 nt]. */
int shine_mesh_clusters(const float* verts, int64_t nv, const int32_t* tris, int64_t nt, int32_t min_tris,
                        void* edge_slots, uint32_t edge_capacity, int32_t* scratch, uint8_t* keep, float* normals,
                        void* stream);

/* ---- evaluation: eval/eval_utils.py eval_mesh / crop_intersection ----------------------------------------------------
 * Uniform sampling of a mesh (Open3D SamplePointsUniformly) in two calls, with one host read between them:
 *   areas: area_t = 0.5 |(p0 - p1) x (p0 - p2)| in fp64 for every triangle, 0 for a triangle with a vertex outside
 *     crop_box (device [6] fp64: min x y z, max x y z, inclusive; NULL = no crop); their inclusive prefix sums, by a
 *     deterministic chunked scan, in the scratch; the total area S to the device double *total_area.
 *   points: sample k lies on the first triangle t with round(cum_t / S * N) > k (N for the last triangle), at
 *     (a v0 + b v1) + c v2 in fp64 with a = 1 - sqrt(r1), b = sqrt(r1)(1 - r2), c = sqrt(r1) r2; (r1, r2) are two 53-bit
 *     doubles in [0, 1) from Philox4x32-10 with key seed and counter k.  S must be > 0 when num_samples > 0.
 *     tri_ids [N] (optional) receives t.
 * Vertices are fp64 [num_verts, 3]; triangles int32 [num_tris, 3] with indices in [0, num_verts). */
int64_t shine_mesh_sample_scratch_bytes(int64_t num_tris);
int shine_mesh_sample_areas(const double* verts, int64_t num_verts, const int32_t* tris, int64_t num_tris,
                            const double* crop_box, double* total_area, void* scratch, int64_t scratch_bytes,
                            void* stream);
int shine_mesh_sample_points(const double* verts, const int32_t* tris, int64_t num_tris, const double* total_area,
                             int64_t num_samples, uint64_t seed, const void* scratch, int64_t scratch_bytes,
                             double* points, int32_t* tri_ids, void* stream);

/* Exact nearest neighbour within a radius.  build: a tree over n fp64 reference points [n, 3] in the caller's `tree`
 * buffer (shine_nn_tree_bytes(n), kept until the last query; 256-byte aligned).  query: for each of m fp64 points,
 * d2 = (dx*dx + dy*dy) + dz*dz (no contraction) minimised over the reference points; if d2 < radius2, dist = sqrt(d2)
 * and index = the input index of a nearest point (any one of exact ties), else dist = +inf and index = -1.
 * scratch: shine_nn_scratch_bytes(n) for a build, shine_nn_scratch_bytes(m) for a query, 256-byte aligned. */
int64_t shine_nn_tree_bytes(int64_t n);
int64_t shine_nn_scratch_bytes(int64_t n);
int shine_nn_build(const double* points, int64_t n, void* tree, int64_t tree_bytes, void* scratch, int64_t scratch_bytes,
                   void* stream);
int shine_nn_query(const void* tree, int64_t n, const double* queries, int64_t m, double radius2, double* dist,
                   int32_t* index, void* scratch, int64_t scratch_bytes, void* stream);

/* ---- scan-to-map registration: one Gauss-Newton system of a scan against the SDF map (odometry.py) ------------------
 * For every point p_i of points (device fp32 [n,3], sensor frame, scaled coordinates) and the pose T (host fp64, 4x4
 * row-major, translation scaled; row 3 is not read), with R and t rounded to fp32:
 *   q = R p + t              fp32, per row ((R0 x + R1 y) + R2 z) + t, every operation rounded on its own;
 *   r = sigma pred(q)        pred as shine_sdf_infer computes it (fp32 FMA chains here), sigma = sigma_sigmoid: the SDF;
 *   g = sigma dpred/dq       back through the ReLU masks to the feature, then through the blend weights
 *                            (shine_query_coord_grad's derivatives);
 *   valid                    q's voxel exists at lv[0]; other points contribute nothing;
 *   Jr = [g, q x g]          the Jacobian of r for a left-multiplied twist (rho, phi), in fp64 from the fp32 q and g;
 *   w = (k^2 / (k^2 + r^2))^2  Geman-McClure weight in fp64, k = kappa (scaled units).
 * out (device fp64 [SHINE_REGISTER_OUT]) = the 21 entries of sum w Jr^T Jr (upper triangle, row-major: (0,0), (0,1) ..
 * (0,5), (1,1) ..), the 6 of sum w Jr^T r, sum w r^2 and the number of valid points.  Per-thread fp64 sums, block
 * partials into scratch (device, 8-byte aligned, >= SHINE_REGISTER_SCRATCH_BYTES), a second launch adds them in a fixed
 * order: the result does not change from run to run.  n = 0 writes zeros.  NULL pointers, n < 0, a non-positive or
 * non-finite kappa or sigma, a non-finite pose entry and a short scratch are SHINE_ERR_INVALID_ARG; a decoder other than
 * 8 -> 32 -> 32 -> 1 is SHINE_ERR_UNSUPPORTED; none of them launches. */
#define SHINE_REGISTER_OUT 29
#define SHINE_REGISTER_MAX_BLOCKS 1024
#define SHINE_REGISTER_SCRATCH_BYTES (SHINE_REGISTER_MAX_BLOCKS * SHINE_REGISTER_OUT * 8)
int shine_register_normal_eq(const shine_octree* oct, const shine_decoder* dec, const float* points, int64_t n,
                             const double* pose, float sigma, double kappa, double* out, void* scratch,
                             int64_t scratch_bytes, void* stream);

/* The same normal equations at num_poses poses of one scan (a grid search, several Gauss-Newton starts): poses is host
 * fp64 [num_poses, 16] (each as pose above), out device fp64 [num_poses, SHINE_REGISTER_OUT].  Row k equals, bit for
 * bit, what shine_register_normal_eq returns at pose k: the same per-point work, block count and fold order, with the
 * pose as the grid's second dimension.  scratch (device, 8-byte aligned) holds every pose's block partials:
 * shine_register_scratch_bytes(n, num_poses) bytes, that is min(ceil(n / 256), SHINE_REGISTER_MAX_BLOCKS) * num_poses *
 * SHINE_REGISTER_OUT * 8.  num_poses <= 0 or above INT32_MAX, a NULL poses or out, a non-finite entry of any pose, a short
 * scratch and the checks of shine_register_normal_eq are refused as there, before any launch.  shine_register_scratch_bytes
 * returns -1 for n < 0 or such a num_poses. */
int64_t shine_register_scratch_bytes(int64_t n, int64_t num_poses);
int shine_register_normal_eq_poses(const shine_octree* oct, const shine_decoder* dec, const float* points, int64_t n,
                                   const double* poses, int64_t num_poses, float sigma, double kappa, double* out,
                                   void* scratch, int64_t scratch_bytes, void* stream);

/* The same normal equations for num_items items of many scans at once (scans localized in lock-step): points is one
 * device fp32 [num_points, 3] array holding every scan, item k is the segment points[seg_begin[k] .. seg_begin[k] +
 * seg_n[k]) at the pose poses[16 k ..] (host fp64, as above), and out (device fp64 [num_items, SHINE_REGISTER_OUT]) row k
 * equals, bit for bit, shine_register_normal_eq(points + 3 seg_begin[k], seg_n[k], pose k): item k runs its own
 * G_k = min(ceil(n_k / 256), SHINE_REGISTER_MAX_BLOCKS) blocks with its own grid-stride, its partials sit at its own
 * prefix offset of the scratch and its fold adds them in block order.  Items may share a segment; an empty segment gives
 * a row of zeros.  seg_begin and seg_n are host int64 [num_items]; the items go to the device in the kernel parameters,
 * at most SHINE_REGISTER_ITEMS_PER_LAUNCH per launch.  scratch (device, 8-byte aligned) holds
 * shine_register_scans_scratch_bytes(seg_n, num_items) = sum_k G_k * SHINE_REGISTER_OUT * 8 bytes.  Everything
 * shine_register_normal_eq_poses refuses (with num_points as n), a NULL seg_begin or seg_n, a negative seg_n[k] or
 * seg_begin[k], and a segment reaching past num_points are SHINE_ERR_INVALID_ARG, before any launch.
 * shine_register_scans_scratch_bytes returns -1 for a NULL seg_n, a negative entry, or num_items <= 0 or above
 * INT32_MAX. */
#define SHINE_REGISTER_ITEMS_PER_LAUNCH 384
int64_t shine_register_scans_scratch_bytes(const int64_t* seg_n, int64_t num_items);
int shine_register_normal_eq_scans(const shine_octree* oct, const shine_decoder* dec, const float* points,
                                   int64_t num_points, const int64_t* seg_begin, const int64_t* seg_n,
                                   const double* poses, int64_t num_items, float sigma, double kappa, double* out,
                                   void* scratch, int64_t scratch_bytes, void* stream);

/* ---- ray casting: where rays from one sensor origin first meet the map's zero level set (evaluate.py eval_scans) ----
 * Ray i goes from origin (host fp32 [3], scaled) towards points[i] (device fp32 [n,3], scaled, map frame).  fp32, every
 * operation rounded on its own: v = p - o, r = sqrt((vx vx + vy vy) + vz vz), d = v / r, and the lattice
 *   t_k = t_min + k h,  x_k = o + t_k d,  k = 0 .. K,  K = min(floor((min(r + beyond, t_max) - t_min) / h), 2^24 - 1)
 * (no sample when K < 0, or r is 0 or not finite).  At each sample m_k = x_k's voxel exists at lv[mask_level] and
 * s_k = -Decoder.sdf(f(x_k)): the value and mask of shine_mesh_grid (positive in free space, the mesher's mask), here
 * with an fp32 FMA blend and decoder.  The hit is the first k >= 1 with m_{k-1}, m_k, s_{k-1} > 0 and s_k <= 0; at most
 * refine_iters bisection steps follow, t_mid = 0.5 (t_a + t_b), ending early when t_mid is not strictly inside the bracket
 * or x(t_mid) is masked; out_t[i] = t_a + (t_b - t_a) (s_a / (s_a - s_b)) over the final bracket, the hit distance in
 * scaled units, and out_status[i] = 1.  A miss: out_t[i] = NaN, out_status[i] = 0.  Samples whose cell at the coarsest
 * featured level holds no node are skipped, with the same result as a march over every sample.  One thread per ray, no
 * atomics: two launches on the same inputs give the same bits.  n < 0, NULL buffers (n > 0), a non-finite origin, h not
 * finite and > 0, a non-finite t_min, t_max <= t_min, beyond < 0 or not finite, refine_iters outside
 * [0, SHINE_RAYCAST_MAX_REFINE] and mask_level outside [0, num_levels) are SHINE_ERR_INVALID_ARG; a decoder other than
 * 8 -> 32 -> 32 -> 1 is SHINE_ERR_UNSUPPORTED; none of them launches. */
#define SHINE_RAYCAST_MAX_REFINE 32
int shine_raycast(const shine_octree* oct, const shine_decoder* dec, const float* origin, const float* points, int64_t n,
                  float h, float t_min, float beyond, float t_max, int32_t refine_iters, int32_t mask_level,
                  float* out_t, uint8_t* out_status, void* stream);

/* ---- rendering: depth, range and normal images of one camera view of the map (render.py) ----------------------------
 * One ray per pixel (u, v), u = 0 .. width - 1 (column), v = 0 .. height - 1 (row), pixel i = v width + u.  fp32, every
 * operation rounded on its own.  The camera-frame unit direction c:
 *   SHINE_CAMERA_PINHOLE:     a = (u - cx) / fx,  b = (v - cy) / fy,  n = sqrt((a a + b b) + 1),  c = (a / n, b / n, 1 / n)
 *                             (the pixel centre is (u, v), as shine_rgbd_backproject); depth = t c_z.
 *   SHINE_CAMERA_RANGE_IMAGE: el = el0 - v del,  az = az0 - u daz  (fp32), with, in fp64 rounded once to fp32,
 *                             el0 = fov_up pi / 180, del = (fov_up - fov_down) pi / 180 / (height - 1) (0 when height = 1),
 *                             az0 = pi, daz = 2 pi / width: row 0 looks at fov_up, the last row at fov_down, column 0 at
 *                             azimuth +pi and the azimuth falls with the column.  ce, se, ca, sa = cos and sin of el and az,
 *                             each evaluated in fp64 and rounded to fp32; c = (ce ca, ce sa, se); depth = t.
 * pose (host fp32 [12]) is the 3x4 camera-to-map transform, row-major, in scaled map coordinates: the ray's direction is
 * d = R c, per row ((R0 c0 + R1 c1) + R2 c2), and its origin o the translation.  Along the ray the lattice and the march
 * are shine_raycast's, with K = min(floor((t_max - t_min) / h), 2^24 - 1) for every pixel (no per-ray endpoint, no beyond).
 * Outputs (device, NULL: not wanted): out_range [H W] = the hit distance t in scaled units, out_depth [H W] as above,
 * out_normal [H W 3] = -g / |g| with g = dpred/dq at the hit point x = o + t d (fp32, shine_raycast's sample rounding): the
 * gradient shine_register_normal_eq forms without sigma, back through the ReLU masks and the blend weights, so that
 * n is the unit gradient of the march's field -Decoder.sdf (it faces free space); |n| = sqrt((gx gx + gy gy) + gz gz),
 * then each component is -(g_a / |g|).  out_status [H W] = 1 on a hit.  A miss: NaN range, depth and normal, status 0.
 * One thread per pixel, no atomics: two launches on the same inputs give the same bits.  NULL cam or pose, width or
 * height <= 0, width height > 2^31, a non-finite pose entry, an unknown model, a pinhole with non-finite intrinsics or
 * fx, fy <= 0, a range image with a non-finite FOV or fov_up <= fov_down, a non-finite t_max and shine_raycast's checks of
 * h, t_min, t_max, refine_iters and mask_level are SHINE_ERR_INVALID_ARG; a decoder other than 8 -> 32 -> 32 -> 1 is
 * SHINE_ERR_UNSUPPORTED; none of them launches.  No wanted output: SHINE_OK without a launch. */
#define SHINE_CAMERA_PINHOLE 0
#define SHINE_CAMERA_RANGE_IMAGE 1
typedef struct shine_camera {
    int32_t model;              /* SHINE_CAMERA_PINHOLE or SHINE_CAMERA_RANGE_IMAGE */
    int32_t width, height;      /* pixels */
    float fx, fy, cx, cy;       /* pinhole, pixels */
    float fov_up, fov_down;     /* range image, degrees */
} shine_camera;
int shine_render(const shine_octree* oct, const shine_decoder* dec, const shine_camera* cam, const float* pose, float h,
                 float t_min, float t_max, int32_t refine_iters, int32_t mask_level, float* out_range, float* out_depth,
                 float* out_normal, uint8_t* out_status, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SHINE_B200_H_ */
