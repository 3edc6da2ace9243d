/* include/detable.h -- C ABI of the H100-native (sm_90a) dynamic-embedding table engine.
 *
 * This is the drop-in boundary for the ONE hot path this repo accelerates: the
 * `tfra.dynamic_embedding` table path of tensorflow/recommenders-addons.  Each entry point
 * replaces one method of the reference's table objects, i.e. what the TF custom-op kernels
 * `TFRA>CuckooHashTable*` / `TFRA>HkvHashTable*` call after unpacking their tensors.
 * Reference paths below are relative to
 *   /root/reference/tensorflow_recommenders_addons/dynamic_embedding/core/
 *
 * Conventions
 *   - plain C: pointers + sizes, no torch / TF types.  `det_stream_t` is a `cudaStream_t`.
 *   - unless a parameter says HOST, every data pointer is a DEVICE pointer on the table's GPU.
 *   - every call is asynchronous on the caller's stream and never synchronises, except:
 *       det_size / det_export (return a count to the host), the *_host entry points, and a
 *       mutating call that has to GROW the table (rare; see DESIGN.md "capacity").
 *   - return value: DET_OK or an error code; det_last_error() gives the message of the last
 *     failing call on the calling thread (mirrors OP_REQUIRES_OK(ctx, Status),
 *     kernels/cuckoo_hashtable_op.cc:601-604; HKV exceptions -> Status(kInternal),
 *     kernels/lookup_impl/lookup_table_op_hkv.h:54-60).
 *   - keys are int64 (the only key type the reference registers on GPU,
 *     kernels/hkv_hashtable_op_gpu.cu.cc:1133-1138); ALL 2^64 key values are legal.
 *   - rows are `dim` elements of `value_dtype`, contiguous, row-major [n, dim].
 *   - keys inside ONE mutating call must be unique (same contract as the reference's GPU
 *     table, python/ops/dynamic_embedding_variable.py:1377-1378).  Duplicates are memory-safe:
 *     the key is stored once; insert keeps one of the rows per 16-byte chunk, accum adds all.
 *   - concurrency (the reference serialises every op on one table with a reader/writer mutex,
 *     kernels/hkv_hashtable_op_gpu.cu.cc:201,258; here calls are stream-ordered instead):
 *       * calls on ONE stream see each other's effects in issue order;
 *       * read-only calls (det_find, det_find_scores, det_lookup_sparse, det_peer_find) may run
 *         concurrently on any streams / host threads, also while another host thread grows the
 *         table (det_find holds a shared host lock against the plane swap);
 *       * a read-only call and a mutating call that overlap in time on DIFFERENT streams (e.g.
 *         det_find_host_async + det_insert_host_async) are only defined for DISJOINT key sets:
 *         a row being rewritten may be read torn (16-byte chunks of the old and new row), keys
 *         are never torn and no other key is affected;
 *       * two mutating calls on one table must be stream-ordered (host bookkeeping is
 *         serialised by a per-table mutex, device work is not).
 */
#ifndef DETABLE_H_
#define DETABLE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct det_table det_table;
typedef void* det_stream_t; /* cudaStream_t */
typedef int det_status;

enum {
  DET_OK = 0,
  DET_INVALID_ARGUMENT = 1, /* errors::InvalidArgument */
  DET_OUT_OF_MEMORY = 2,    /* "...adjust param 'max_hbm' smaller", lookup_table_op_hkv.h:364-368 */
  DET_CUDA_ERROR = 3,       /* CUDA_CHECK */
  DET_TABLE_FULL = 4,       /* max_capacity reached */
  DET_UNIMPLEMENTED = 5,
  DET_INTERNAL = 6,
  DET_IO_ERROR = 7
};

/* value dtypes the reference registers for its GPU table (hkv_hashtable_op_gpu.cu.cc:1133-1138) */
enum {
  DET_FLOAT32 = 0,
  DET_FLOAT16 = 1,
  DET_BFLOAT16 = 2,
  DET_INT32 = 3,
  DET_INT64 = 4,
  DET_INT8 = 5,
  DET_FLOAT64 = 6
};

/* combiner of embedding_lookup_sparse (python/ops/dynamic_embedding_ops.py:205-206) */
enum { DET_COMBINER_SUM = 0, DET_COMBINER_MEAN = 1, DET_COMBINER_SQRTN = 2 };

/* Attributes of the table-creating ops:
 *   CuckooHashTableOfTensors: key_dtype, value_dtype, value_shape, init_size  (ops/cuckoo_hashtable_ops.cc:293-309)
 *   HkvHashTableOfTensors:    + init_capacity, max_capacity, ...              (ops/hkv_hashtable_ops.cc:318-331) */
typedef struct det_config {
  int32_t value_dtype;      /* DET_FLOAT32 ... */
  int32_t dim;              /* value_shape[0] */
  int32_t device;           /* CUDA device ordinal */
  int32_t num_slot_planes;  /* 0..3 optimizer slot planes co-indexed with the value rows: fp32 rows of 4 * dim bytes
                             * beside DET_FLOAT32, DET_FLOAT16 or DET_BFLOAT16 value rows (other dtypes: 0 only); with
                             * DET_FLAGS_SLOTS_IN_VALUE_DTYPE on a DET_FLOAT16 / DET_BFLOAT16 table, rows of that dtype
                             * (2 * dim bytes) */
  uint64_t init_capacity;   /* keys; 0 -> 8192 (TF_HASHTABLE_INIT_SIZE default, cuckoo_hashtable_op.cc:199-205) */
  uint64_t max_capacity;    /* SLOTS (HKV's max_capacity); 0 -> grow without bound (cuckoo semantics); else the table
                             * holds at most max_load_factor * max_capacity keys and answers DET_TABLE_FULL beyond */
  float max_load_factor;    /* 0 -> 0.75 (0.875 with an eviction strategy) */
  uint32_t flags;           /* bits 0..3: eviction strategy + 1 (DET_FLAGS_EVICT), 0 = none; bit 4:
                             * DET_FLAGS_SLOTS_IN_VALUE_DTYPE; other bits reserved, 0 */
  uint64_t max_hbm_for_vectors; /* ABI >= 3.  Bytes of HBM the VALUE rows may take (attr `max_hbm_for_vectors`,
                             * ops/hkv_hashtable_ops.cc:318-331 -> HashTableOptions, lookup_table_op_hkv.h:443-448);
                             * 0 = all rows in HBM.  Rows beyond the budget live in pinned HOST memory that the
                             * same kernels reach over PCIe (one virtual range, DESIGN.md 4c); keys, scores and
                             * optimizer slot planes always stay in HBM.  Ignored by tables in a caller's region. */
} det_config;

/* Eviction strategies of the HKV table (python/ops/hkv_hashtable_ops.py HkvEvictStrategy; kernels/lookup_impl/
 * lookup_table_op_hkv.h:454-479).  With a strategy the table keeps a uint64 SCORE per key and, once it holds
 * max_load_factor * max_capacity keys, evicts the lowest-scored keys to make room instead of failing with
 * DET_TABLE_FULL (DESIGN.md "capacity management"); with max_capacity == 0 it keeps the scores, grows without
 * bound and only det_evict removes keys.  Score of a key after insert / assign / accum:
 *   LRU  device clock (ns)      EPOCHLRU  epoch << 32 | low32(clock >> 20)
 *   LFU  old + delta            EPOCHLFU  epoch << 32 | min(low32(old) + delta, 2^32 - 1)     (delta: `scores`, default 1)
 *   CUSTOMIZED  the score the caller provides. */
enum {
  DET_EVICT_NONE = -1,
  DET_EVICT_LRU = 0,
  DET_EVICT_LFU = 1,
  DET_EVICT_EPOCHLRU = 2,
  DET_EVICT_EPOCHLFU = 3,
  DET_EVICT_CUSTOMIZED = 4
};
#define DET_FLAGS_EVICT(strategy) ((uint32_t)((strategy) + 1) & 0xFu)

/* Optimizer slot planes in the table's own value dtype (the layout of the reference, whose slot Variables take the
 * param's value_dtype, python/ops/dynamic_embedding_optimizer.py:889-901).  On a DET_FLOAT16 / DET_BFLOAT16 table every
 * slot plane holds rows of that dtype, 2 * dim bytes; on a DET_FLOAT32 table the flag changes nothing.  The fused step
 * widens each slot element to fp32 (exact), runs the fp32 rule, and rounds every slot value it writes to nearest even
 * into the dtype once, at its store, as it does the param; the new param comes from the unrounded fp32 slot values.  A
 * slot without state (a key the step creates, or one written by insert / accum and never stepped) starts from its
 * initial value rounded into the dtype.  fp32 planes stay the default: a half accumulator loses small updates (an fp16
 * Adagrad accumulator drops g*g below |g| ~ 1.7e-4, DESIGN.md section 4).  det_table_create_in_region and the
 * det_peer_* groups refuse a table with the flag (DET_UNIMPLEMENTED).  Additive to ABI 8. */
#define DET_FLAGS_SLOTS_IN_VALUE_DTYPE (1u << 4)

/* ---- lifetime: HashTableOp::Compute / LookupOrCreate, kernels/cuckoo_hashtable_op.h:59-110 ---- */
det_status det_table_create(det_table** out, const det_config* cfg);
det_status det_table_destroy(det_table* t);
/* A table inside caller-provided device memory (fixed capacity = cfg->init_capacity slots, never grows, memory not
 * freed by destroy): lets the planes live in memory that peers map, see det_peer_group_create_regions.  With
 * DET_FLAGS_EVICT in cfg->flags the table evicts in place at that capacity (the score plane is the library's own). */
size_t det_table_region_bytes(const det_config* cfg);
det_status det_table_create_in_region(det_table** out, const det_config* cfg, void* region, size_t region_bytes);
const char* det_last_error(void);
/* library/ABI probe used by the loaders */
int det_abi_version(void);
const char* det_build_info(void);

/* Keyed random initializer: the row of a missing key is a pure function of (seed, key, column), computed by the kernels
 * where they find the key missing.  Element j of the row of key k: x = Philox4x32-10(counter = (lo32 k, hi32 k, j >> 2,
 * 0), key = (lo32 seed, hi32 seed))[j & 3], u = ((x >> 8) | 1) * 2^-24, then
 *   DET_INIT_UNIFORM           u * (b - a) + a                                   (a, b) = (minval, maxval)
 *   DET_INIT_NORMAL            sqrt(2) * erfinv(2u - 1) * b + a                   (a, b) = (mean, stddev)
 *   DET_INIT_TRUNCATED_NORMAL  sqrt(2) * erfinv(erf(sqrt 2) * (2u - 1)) * b + a   (the law of N(a, b) inside a +- 2b)
 * in fp32 (erfinv: Giles' single-precision approximation), rounded to nearest even into the table's dtype.  The row does
 * not depend on the batch, call order, capacity or device.  With an initializer set, a NULL row pointer means "generate"
 * in det_find (defaults, full_size_default 0), det_lookup_sparse(_clip) (default_row), det_apply_* (init_param,
 * full_size_init 0) and det_apply_*_dup (init_param); without one NULL stays DET_INVALID_ARGUMENT.  The host-buffer
 * finds and the det_peer_* calls do not generate rows.  Float32, float16 and bfloat16 tables; `init` NULL clears. */
enum { DET_INIT_UNIFORM = 1, DET_INIT_NORMAL = 2, DET_INIT_TRUNCATED_NORMAL = 3 };
typedef struct det_initializer {
  int32_t kind;
  int32_t reserved;
  uint64_t seed;
  float a, b;
} det_initializer;
det_status det_table_set_initializer(det_table* t, const det_initializer* init);

/* ---- LookupInterface surface (kernels/cuckoo_hashtable_op.cc:211-308; GPU twin
 *      kernels/hkv_hashtable_op_gpu.cu.cc:181-470) ---- */

/* Find / FindWithExists (cuckoo_hashtable_op.cc:215-233; TableWrapperOptimized::find,
 * kernels/lookup_impl/lookup_table_op_cpu.h:188-217).  A missing key yields the default row:
 * defaults[i,:] if full_size_default else defaults[0,:] (is_full_default rule, :48-50).
 * `exists` may be NULL.  Lookup never inserts. */
det_status det_find(det_table* t, const int64_t* keys, size_t n, const void* defaults,
                    int full_size_default, void* values_out, uint8_t* exists, det_stream_t stream);

/* Insert = insert_or_assign per key (cuckoo_hashtable_op.cc:235-266; lookup_table_op_cpu.h:165-171). */
det_status det_insert(det_table* t, const int64_t* keys, const void* values, size_t n,
                      det_stream_t stream);

/* Accum = insert_or_accum (cuckoo_hashtable_op.cc:248-286; lib/cuckoo/cuckoohash_map.hh:620-633):
 *   found & exists[i] -> row += values_or_deltas[i];  !found & !exists[i] -> insert row;  else no-op. */
det_status det_accum(det_table* t, const int64_t* keys, const void* values_or_deltas,
                     const uint8_t* exists, size_t n, det_stream_t stream);

/* Remove (cuckoo_hashtable_op.cc:268-276): absent keys are ignored. */
det_status det_remove(det_table* t, const int64_t* keys, size_t n, det_stream_t stream);

/* Clear (cuckoo_hashtable_op.cc:278-281). */
det_status det_clear(det_table* t, det_stream_t stream);

/* size() (cuckoo_hashtable_op.cc:213).  HOST out; synchronises `stream`. */
det_status det_size(det_table* t, int64_t* size_out_host, det_stream_t stream);

/* capacity in keys at the current allocation (lookup_table_op_hkv.h:750). No sync. */
det_status det_capacity(det_table* t, uint64_t* capacity_out_host);

/* Make room for `total_keys` keys without further growth (cuckoohash_map::reserve). May sync. */
det_status det_reserve(det_table* t, uint64_t total_keys, det_stream_t stream);

/* ExportValues (cuckoo_hashtable_op.cc:293-308): writes up to max_n (key,row) pairs in table order,
 * *n_out_host = number written (HOST).  plane = 0 value rows, 1..num_slot_planes an optimizer slot
 * plane (the reference keeps each slot in its own table `<var>/<opt>/<slot>`,
 * python/ops/dynamic_embedding_optimizer.py:870-958) in the plane's dtype (fp32, or the table's dtype with
 * DET_FLAGS_SLOTS_IN_VALUE_DTYPE); a slot row that was never stepped reads as the slot's initial value (rounded into the
 * plane's dtype).  Synchronises `stream`. */
det_status det_export(det_table* t, int plane, int64_t* keys_out, void* values_out, size_t max_n,
                      int64_t* n_out_host, det_stream_t stream);

/* The same export restricted to the window [first, first + max_n) of the table order: *n_out_host = rows written
 * (0 once `first` is past the end).  HKV's `dump(keys, values, offset, search_length, counter)` /
 * `export_batch` (lookup_table_op_hkv.h:550-594) -- lets a caller stream a table larger than its scratch memory
 * (det_save does).  The table must not be mutated between the windows of one pass.  ABI >= 3. */
det_status det_export_window(det_table* t, int plane, uint64_t first, int64_t* keys_out, void* values_out,
                             size_t max_n, int64_t* n_out_host, det_stream_t stream);

/* ImportValues = clear + insert (cuckoo_hashtable_op.cc:288-291). */
det_status det_import(det_table* t, const int64_t* keys, const void* values, size_t n,
                      det_stream_t stream);

/* ---- tables with an eviction strategy: the `scores` input of the HKV ops (ops/hkv_hashtable_ops.cc:191-219),
 * ExportWithScores / ExportKeysAndScores (:259-294), set_global_epoch (lookup_table_op_hkv.h:499-507) ----
 * det_insert / det_accum / det_apply_* on such a table behave as if scores == NULL.
 * scores: DEVICE uint64[n] or NULL.  A key that is not in the table is refused (not inserted) when the table is at
 * its limit and the key's score is below every resident score (HKV: below its bucket's minimum). */
det_status det_insert_scored(det_table* t, const int64_t* keys, const void* values, const uint64_t* scores, size_t n,
                             det_stream_t stream);
det_status det_accum_scored(det_table* t, const int64_t* keys, const void* values_or_deltas, const uint8_t* exists,
                            const uint64_t* scores, size_t n, det_stream_t stream);
/* scores_out[i] = score of keys[i], 0 when absent (export_with_scores = det_export + det_find_scores of its keys) */
det_status det_find_scores(det_table* t, const int64_t* keys, size_t n, uint64_t* scores_out, det_stream_t stream);
det_status det_set_global_epoch(det_table* t, uint64_t epoch);
/* Evict the n_evict lowest-scored keys now (what the reference's restrict policies do with a side table and a
 * top-k, python/ops/restrict_policies.py:118-361).  *n_evicted_out_host may be NULL.  Synchronises `stream`. */
det_status det_evict(det_table* t, uint64_t n_evict, int64_t* n_evicted_out_host, det_stream_t stream);

/* ---- fused entry points (replace chains of reference ops; SURVEY.md 2b K6/K7) ---- */

/* tf.unique as used by embedding_lookup_sparse / embedding_lookup_unique
 * (python/ops/dynamic_embedding_ops.py:224, :95): unique_out in first-occurrence order,
 * idx_out[i] = position of ids[i] in unique_out, *n_unique_dev (DEVICE int64).
 * workspace: det_unique_workspace_bytes(n) bytes of device scratch. */
size_t det_unique_workspace_bytes(size_t n);
det_status det_unique(const int64_t* ids, size_t n, int64_t* unique_out, int32_t* idx_out,
                      int64_t* n_unique_dev, void* workspace, size_t workspace_bytes,
                      det_stream_t stream);

/* Gradient dedupe of the sparse optimizer path: out[g, :] = sum of rows[i, :] over the positions i with idx[i] == g,
 * added in INCREASING POSITION (the order of TF's CPU unsorted_segment_sum, which _deduplicate_indexed_slices applies
 * before _resource_apply_sparse_duplicate_indices, python/ops/dynamic_embedding_optimizer.py:150,184; the gradient of
 * dynamic_stitch / sparse_segment_sum, python/ops/data_flow_grad.py:65, python/ops/math_grad.py:30) -- deterministic and
 * bit-identical to np.add.at, where atomics would make the fp32 sum depend on the schedule.  idx is what det_unique
 * returns; indices outside [0, n_groups) are dropped; groups without rows come out as zeros.  rows fp32 [n, dim],
 * out fp32 [n_groups, dim] (every row is written).  workspace: det_segment_reduce_workspace_bytes(n, n_groups) bytes
 * of device scratch.  Asynchronous on `stream`, no host synchronisation.  ABI >= 4. */
size_t det_segment_reduce_workspace_bytes(size_t n, size_t n_groups);
det_status det_segment_reduce(const float* rows, const int32_t* idx, size_t n, size_t n_groups, size_t dim,
                              float* out, void* workspace, size_t workspace_bytes, det_stream_t stream);

/* The tail of embedding_lookup_sparse when the unique rows are a DENSE matrix (training: the TrainableWrapper's scratch,
 * python/ops/dynamic_embedding_ops.py:247-289 -- gather(embeddings, idx) * weights -> segment_sum -> normalise; TF's
 * sparse_segment_sum / mean / sqrt_n): out[b] = combine_{i in segment b} weights[i] * rows[row_idx[i]], the ids of a
 * segment added in order (same arithmetic and kernels as det_lookup_sparse's second phase; the [nnz, dim] gather is
 * never materialised).  rows fp32 [n_rows, dim]; row_idx int64 [nnz] (the idx of det_unique, widened; < 0 reads
 * default_row [dim]); segment_ids int32 [nnz] ascending in [0, batch); weights [nnz] or NULL; out fp32 [batch, dim].
 * Indices must lie in [.., n_rows): they are not checked.  workspace: det_sparse_segment_sum_workspace_bytes(batch).
 * Asynchronous on `stream`.  ABI >= 4. */
size_t det_sparse_segment_sum_workspace_bytes(size_t batch);
det_status det_sparse_segment_sum(const float* rows, size_t dim, const int64_t* row_idx, const int32_t* segment_ids,
                                  const float* weights, size_t nnz, size_t batch, int combiner, const float* default_row,
                                  float* out, void* workspace, size_t workspace_bytes, det_stream_t stream);

/* embedding_lookup_sparse forward, fused (python/ops/dynamic_embedding_ops.py:219-291): a slot-resolve pass
 * (8 B per id) + ONE gather/weight/segment-sum/normalise pass -- the reference's [nnz, dim] gather, its weighted
 * copy and the segment_sum input are never materialised:
 * out[b,:] = combine_{i in segment b} w_i * row(ids[i]); missing ids use `default_row` [dim]
 * (broadcast default).  segment_ids are sorted ascending (canonical SparseTensor order);
 * weights may be NULL (all 1).  Rows of `out` without ids are zero.  Tables of DET_FLOAT32, DET_FLOAT16 or
 * DET_BFLOAT16 rows (DET_UNIMPLEMENTED for the other dtypes); fp16 / bf16 rows are widened to fp32 as they are read
 * (exact), so the result is bit-identical to an fp32 table holding the widened rows.  `default_row`, `weights` and `out`
 * are fp32 whatever the table's dtype, and default_row is used exactly as given: for the reference's result (which casts
 * the looked-up rows, defaults included, to fp32) pass the table's default row widened to fp32.
 * Uses the table's scratch buffer: one stream per table at a time. */
det_status det_lookup_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                             const float* weights, size_t nnz, size_t batch, int combiner,
                             const float* default_row, float* out, det_stream_t stream);

/* The same with `max_norm` (embedding_lookup_sparse(..., max_norm); tf.clip_by_norm of every looked-up row BEFORE it is
 * weighted, python/ops/embedding_weights.py:497-521): row <- row * max_norm / max(||row||_2, max_norm), folded into the
 * gather.  max_norm == 0: no clipping (= det_lookup_sparse).  Rows of at most 32 vectors (dim <= 128 when dim % 4 == 0,
 * else dim <= 32); DET_UNIMPLEMENTED beyond.  max_norm > 0 on a DET_FLOAT16 / DET_BFLOAT16 table is DET_UNIMPLEMENTED:
 * the reference clips in the table's dtype, which a clip folded into the fp32 gather would not reproduce; use the
 * composed path (find, clip, det_sparse_segment_sum).  ABI >= 3. */
det_status det_lookup_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                  const float* weights, size_t nnz, size_t batch, int combiner,
                                  const float* default_row, float max_norm, float* out, det_stream_t stream);

/* safe_embedding_lookup_sparse forward, fused (python/ops/dynamic_embedding_ops.py:296-438; ABI >= 8).  The inputs are
 * the RAW sparse ids: ids int64[nnz], segment_ids int32[nnz] = the flattened row of every entry (for ids of rank r >= 2,
 * row = sum_k idx[:, k] * stride_k over the leading r - 1 dims; batch = their product), ascending (canonical order),
 * weights f32[nnz] or NULL.  Before the lookup, the list is cleaned on the device, as the reference rewrites it:
 *   prune:  only with weights and combiner != DET_COMBINER_SUM, an entry is kept iff w > 0 (NaN weights are pruned);
 *           a pruned id is not looked up and adds nothing to any denominator;
 *   fill:   a row left without an entry (empty, or all of its entries pruned) gets one entry (default_id, weight 1) at
 *           its row position when has_default_id != 0 -- its output is that id's row, bit for bit;
 *           has_default_id == 0: its output row is +0.0 (no entry is added);
 * then out[b] is det_lookup_sparse of the cleaned list (same arithmetic, default_row and dtype rules).  The cleaned
 * count never leaves the device: no host synchronisation.  Rows of `out` are in the flattened row order (reshape to
 * dense_shape[:-1] + (dim,)).  Malformed segment ids (not ascending, or outside [0, batch)) leave every output row +0.0
 * and raise the table's bad-segment error flag (det_get_stats).  Any dim det_lookup_sparse covers; max_norm:
 * det_lookup_sparse_safe_clip.  Uses
 * the table's scratch buffer: one stream per table at a time. */
det_status det_lookup_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                  size_t nnz, size_t batch, int combiner, int has_default_id, int64_t default_id,
                                  const float* default_row, float* out, det_stream_t stream);
/* The same with `max_norm` (safe_embedding_lookup_sparse(..., max_norm); ABI >= 8): every row of the cleaned list,
 * fill rows included, is clipped as det_lookup_sparse_clip clips it, with the same limits and refusals. */
det_status det_lookup_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                       const float* weights, size_t nnz, size_t batch, int combiner, int has_default_id,
                                       int64_t default_id, const float* default_row, float max_norm, float* out,
                                       det_stream_t stream);

/* One DynamicEmbeddingOptimizer step on unique keys, fused (find param + find slot(s) -> dense
 * rule -> upsert param + upsert slot(s); python/ops/dynamic_embedding_optimizer.py:161-204,
 * python/ops/embedding_weights.py:434-444).  Missing keys start from init_param[dim]
 * (or [n,dim] if full_size_init) and the slot initial value, then get inserted.
 * Adagrad: a += g*g; p -= lr*g/(sqrt(a)+eps)   (eps = 0: TF1 AdagradOptimizer; 1e-7: Keras)
 *   slot plane 1 = accumulator.
 * Adam   : m += (g-m)(1-b1); v += (g*g-v)(1-b2); p -= m*alpha/(sqrt(v)+eps),
 *   alpha = lr*sqrt(1-b2^t)/(1-b1^t) computed by the caller;  plane 1 = m, plane 2 = v.
 * Tables of DET_FLOAT32, DET_FLOAT16 and DET_BFLOAT16 values (other dtypes: DET_UNIMPLEMENTED).  On a half table the
 * stored param is widened to fp32 (exact), stepped by the fp32 rule above, and rounded to nearest even into the table's
 * dtype once (overflow to +-inf, subnormals kept, NaN stays NaN); the slot planes stay fp32, or are rounded the same way
 * into the table's dtype with DET_FLAGS_SLOTS_IN_VALUE_DTYPE.  grads and init_param are fp32 whatever the table's dtype
 * (a half initializer row widened to fp32 is exact). */
det_status det_apply_adagrad(det_table* t, const int64_t* keys, const float* grads, size_t n,
                             float lr, float epsilon, const float* init_param, int full_size_init,
                             float init_accum, det_stream_t stream);
det_status det_apply_adam(det_table* t, const int64_t* keys, const float* grads, size_t n,
                          float alpha, float beta1, float beta2, float epsilon,
                          const float* init_param, int full_size_init, det_stream_t stream);
/* The same step for SGD, momentum and FTRL, each fp32 operation rounded on its own, in the order written (TF's sparse
 * CPU kernels).  Keys, init_param, value dtypes, eviction scores: as det_apply_adagrad.  A key the step creates gets
 * the "no slot state" marker in every slot plane the step does not write, as det_insert gives it.
 * SGD     (momentum == 0): p = p - lr*g;  no slot plane needed.
 * Momentum (TF1 MomentumOptimizer; torch SGD(momentum, dampening=0)): a = a*m + g;  p = p - a*lr, or with nesterov
 *   p = p - ((g*lr) + ((a*m)*lr));  plane 1 = momentum (initial 0).  nesterov with momentum == 0: DET_INVALID_ARGUMENT.
 * FTRL    (learning_rate_power = -0.5): gs = l2_shrinkage > 0 ? g + (2*l2_shrinkage)*p : g;  nn = n + g*g;
 *   z = z + (gs - (((sqrt(nn) - sqrt(n)) / lr) * p));  p = (min(max(z, -l1), l1) - z) / (sqrt(nn)/lr + 2*l2);  n = nn
 *   (p is +0 exactly when |z| <= l1);  plane 1 = accumulator n (initial init_accum), plane 2 = linear z (initial 0).
 *   lr <= 0 or a negative l1, l2, l2_shrinkage or init_accum: DET_INVALID_ARGUMENT.
 * Additive to ABI 8. */
det_status det_apply_sgd(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr, float momentum,
                         int nesterov, const float* init_param, int full_size_init, det_stream_t stream);
det_status det_apply_ftrl(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr, float l1, float l2,
                          float l2_shrinkage, const float* init_param, int full_size_init, float init_accum,
                          det_stream_t stream);
/* The same step for RMSprop and Adadelta; r = 1 - rho, computed once in fp32.  Correctly rounded square roots and one
 * division where TF's CPU kernels multiply by rsqrt (not bit-identical to TF, see DESIGN.md section 4).
 * RMSprop: ms = ms*rho + (g*g)*r;  centered: mg = mg*rho + g*r, d = ms - mg*mg;  else d = ms;
 *   momentum > 0:  mom = mom*momentum + (lr*g) / sqrt(d + eps);  p = p - mom;
 *   momentum == 0: p = p - (lr*g) / (eps_in_sqrt ? sqrt(d + eps) : sqrt(d) + eps).
 *   Planes: 1 = rms (initial init_ms), then mg if centered, then mom if momentum > 0 (initial 0); 1 to 3 planes.
 *   Keras RMSprop: eps_in_sqrt = (momentum > 0), init_ms = 0;  TF1 RMSPropOptimizer: eps_in_sqrt = 1, init_ms = 1.
 *   A negative or NaN momentum, or momentum > 0 with eps_in_sqrt == 0: DET_INVALID_ARGUMENT.
 * Adadelta (TF1 AdadeltaOptimizer, Keras Adadelta): acc = acc*rho + (g*g)*r;  u = (sqrt(au + eps) / sqrt(acc + eps))*g;
 *   p = p - u*lr;  au = au*rho + (u*u)*r.  Plane 1 = accum_grad acc, plane 2 = accum_var au (both initial 0).
 * Additive to ABI 8. */
det_status det_apply_rmsprop(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr, float rho,
                             float momentum, float epsilon, int centered, int eps_in_sqrt, const float* init_param,
                             int full_size_init, float init_ms, det_stream_t stream);
det_status det_apply_adadelta(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr, float rho,
                              float epsilon, const float* init_param, int full_size_init, det_stream_t stream);
/* The same step for Adamax, Nadam, ProximalAdagrad, ProximalGradientDescent and AdagradDA.  r1 = 1 - beta1 and
 * r2 = 1 - beta2 are computed once in fp32; the scalars that depend only on the step are the caller's, in fp32.
 * Adamax (Keras): m = m*beta1 + g*r1;  v = max(v*beta2, |g|);  p = p + nsl*(m / (v + eps)) with nsl = -lr_t and
 *   lr_t = lr / (1 - beta1^t) from the caller.  Plane 1 = m, plane 2 = v (both initial 0).
 * Nadam (Keras): g' = g / omsn;  m = m*beta1 + g*r1;  m' = m / omsx;  mbar = omt*g' + mt1*m';
 *   v = v*beta2 + (g*g)*r2;  v' = v / vden;  p = p + (nlr*mbar) / (sqrt(v') + eps) with nlr = -lr.  The caller computes,
 *   as Keras' _prepare_local: u_t = beta1*(1 - 0.5*0.96^(0.004*t)), u_t1 the same at t + 1, msn = m_cache*u_t,
 *   msx = msn*u_t1, omsn = 1 - msn, omsx = 1 - msx, omt = 1 - u_t, mt1 = u_t1, vden = 1 - beta2^t (m_cache: the product
 *   of the earlier steps' u, 1 before the first).  Plane 1 = m, plane 2 = v (both initial 0).
 * Shrink: S(x, c) = sign(x)*max(|x| - c, 0) (sign(0) = 0).
 * ProximalAdagrad (TF1): a = a + g*g;  eta = lr / sqrt(a);  q = p - g*eta;
 *   p = l1 > 0 ? S(q, eta*l1) / (1 + l2*eta) : q / (1 + l2*eta).  A correctly rounded square root and one division
 *   where TF multiplies by rsqrt (DESIGN.md section 4).  Plane 1 = accumulator (initial init_accum).
 * ProximalGradientDescent (TF1): q = p - g*lr, then the same with eta = lr.  No slot plane; with l1 = l2 = 0 it is
 *   det_apply_sgd bit for bit.
 * AdagradDA (TF1): ga = ga + g;  gg = gg + g*g;  p = ((l1 > 0 ? -S(ga, l1*gs) : -ga) / ((l2*gs)*lr + sqrt(gg)))*lr,
 *   with gs = global_step >= 1, TF1's step on the worker (its global step + 1).  Plane 1 = gradient_accumulator ga
 *   (initial 0), plane 2 = gradient_squared_accumulator gg (initial init_gg).
 * lr <= 0, a negative l1, l2 or initial accumulator (NaN included) of the proximal and DA steps, or global_step < 1:
 * DET_INVALID_ARGUMENT.  Additive to ABI 8. */
det_status det_apply_adamax(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr_t, float beta1,
                            float beta2, float epsilon, const float* init_param, int full_size_init, det_stream_t stream);
det_status det_apply_nadam(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr, float beta1,
                           float beta2, float epsilon, float omsn, float omsx, float omt, float mt1, float vden,
                           const float* init_param, int full_size_init, det_stream_t stream);
det_status det_apply_proximal_adagrad(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr, float l1,
                                      float l2, const float* init_param, int full_size_init, float init_accum,
                                      det_stream_t stream);
det_status det_apply_proximal_sgd(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr, float l1,
                                  float l2, const float* init_param, int full_size_init, det_stream_t stream);
det_status det_apply_adagrad_da(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr, float l1,
                                float l2, int64_t global_step, const float* init_param, int full_size_init,
                                float init_gg, det_stream_t stream);
/* The same step for AdamW (and AMSGrad) and Lion, Keras 3's dense update_step after its _apply_weight_decay.  Each
 * fp32 operation is rounded on its own, in the order written; the step scalars are the caller's, in fp32.
 * Weight decay, first, when weight_decay > 0: p = p - (p*weight_decay)*lr.  weight_decay == 0 skips the line (an inf
 * param stays inf).
 * AdamW: m = m + (g - m)*(1 - beta1);  v = v + (g*g - v)*(1 - beta2);  with amsgrad: vh = max(vh, v), then
 *   p = p - (m*alpha) / (sqrt(vh) + epsilon); without it v takes vh's place.  alpha = lr*sqrt(1 - beta2^t)/(1 - beta1^t)
 *   from the caller, as for det_apply_adam; lr is the decay's.  Plane 1 = m, plane 2 = v, plane 3 = vhat (amsgrad only;
 *   all initial 0).  weight_decay = 0 with amsgrad = 0 is det_apply_adam bit for bit (param, m and v).  Keras' own
 *   IndexedSlices branch rounds m and v in another order (DESIGN.md section 4).
 * Lion: c = m*beta1 + g*r1;  p = p - lr*sign(c);  m = m*beta2 + g*r2, with r1 = 1 - beta1 and r2 = 1 - beta2 computed
 *   once in fp32, sign(+-0) = 0 and sign(NaN) = NaN.  Plane 1 = m (initial 0).
 * A negative or NaN weight_decay, or Lion betas outside [0, 1]: DET_INVALID_ARGUMENT.  Additive to ABI 8. */
det_status det_apply_adamw(det_table* t, const int64_t* keys, const float* grads, size_t n, float alpha, float beta1,
                           float beta2, float epsilon, float lr, float weight_decay, int amsgrad, const float* init_param,
                           int full_size_init, det_stream_t stream);
det_status det_apply_lion(det_table* t, const int64_t* keys, const float* grads, size_t n, float lr, float beta1,
                          float beta2, float weight_decay, const float* init_param, int full_size_init,
                          det_stream_t stream);

/* ---- HOST-buffer entry points (the op placed on host tensors; used for end-to-end timing):
 * pinned or pageable HOST pointers; chunked H2D -> kernel -> D2H pipeline on internal streams;
 * synchronous on return. ---- */
det_status det_find_host(det_table* t, const int64_t* keys_host, size_t n, const void* defaults_host,
                         int full_size_default, void* values_out_host, uint8_t* exists_host);
det_status det_insert_host(det_table* t, const int64_t* keys_host, const void* values_host, size_t n);
/* Asynchronous flavours (PINNED host buffers only): return once everything is enqueued on the table's internal
 * streams; det_host_sync() waits.  Find and insert use separate streams, so a lookup of batch i+1 (D2H-heavy)
 * overlaps the write-back of batch i (H2D-heavy) on a full-duplex PCIe link -- input prefetch as tf.data does. */
det_status det_find_host_async(det_table* t, const int64_t* keys_host, size_t n, const void* defaults_host,
                               int full_size_default, void* values_out_host, uint8_t* exists_host);
det_status det_insert_host_async(det_table* t, const int64_t* keys_host, const void* values_host, size_t n);
det_status det_host_sync(det_table* t);
/* ABI >= 8.  which = 0: everything det_find_host_async has enqueued is on the host; 1: everything det_insert_host_async
 * has enqueued has been applied; -1: both (= det_host_sync).  A loop that prefetches the rows of step i+1 and writes
 * step i back waits with which = 0: the write-back keeps draining while the next step's copies start, so both PCIe
 * directions stay busy across step boundaries. */
det_status det_host_sync_pipe(det_table* t, int which);

/* Sparse apply_gradients with REPEATED ids in ONE call and without host synchronisation (ABI >= 6): what the reference's
 * optimizer patch does for IndexedSlices gradients -- unique(ids) -> unsorted_segment_sum(grads, idx, n_unique) ->
 * find / dense rule / upsert per unique id (python/ops/dynamic_embedding_optimizer.py:150,184 and :161-204) -- as
 * det_unique -> det_segment_reduce (rows of one id added in position order, bit-identical to the sequential sum) ->
 * the fused find-or-insert optimizer kernel, chained on `stream` with the unique count staying ON THE DEVICE.
 * ids int64[n] (repeats allowed), grads f32[n, dim]; new keys start from the broadcast row init_param[dim].
 * workspace: det_apply_dup_workspace_bytes(n, dim) bytes of device memory, 256 B aligned, stream-ordered scratch.
 * n_unique_dev_out (nullable): device int64 that receives the number of distinct ids.
 * DET_UNIMPLEMENTED for rows that are not 16-byte vectors (use det_unique + det_segment_reduce + det_apply_*).
 * Value dtypes and the narrowing of a half table's param: as det_apply_adagrad / det_apply_adam. */
size_t det_apply_dup_workspace_bytes(size_t n, size_t dim);
det_status det_apply_adagrad_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr, float epsilon,
                                 const float* init_param, float init_accum, void* workspace, size_t workspace_bytes,
                                 int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_adam_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float alpha, float beta1,
                              float beta2, float epsilon, const float* init_param, void* workspace,
                              size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_sgd_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr, float momentum,
                             int nesterov, const float* init_param, void* workspace, size_t workspace_bytes,
                             int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_ftrl_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr, float l1,
                              float l2, float l2_shrinkage, const float* init_param, float init_accum, void* workspace,
                              size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_rmsprop_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr, float rho,
                                 float momentum, float epsilon, int centered, int eps_in_sqrt, const float* init_param,
                                 float init_ms, void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                 det_stream_t stream);
det_status det_apply_adadelta_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr, float rho,
                                  float epsilon, const float* init_param, void* workspace, size_t workspace_bytes,
                                  int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_adamax_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr_t, float beta1,
                                float beta2, float epsilon, const float* init_param, void* workspace,
                                size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_nadam_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr, float beta1,
                               float beta2, float epsilon, float omsn, float omsx, float omt, float mt1, float vden,
                               const float* init_param, void* workspace, size_t workspace_bytes,
                               int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_proximal_adagrad_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr,
                                          float l1, float l2, const float* init_param, float init_accum, void* workspace,
                                          size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_proximal_sgd_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr, float l1,
                                      float l2, const float* init_param, void* workspace, size_t workspace_bytes,
                                      int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_adagrad_da_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr, float l1,
                                    float l2, int64_t global_step, const float* init_param, float init_gg,
                                    void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                    det_stream_t stream);
det_status det_apply_adamw_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float alpha, float beta1,
                               float beta2, float epsilon, float lr, float weight_decay, int amsgrad,
                               const float* init_param, void* workspace, size_t workspace_bytes,
                               int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_lion_dup(det_table* t, const int64_t* ids, const float* grads, size_t n, float lr, float beta1,
                              float beta2, float weight_decay, const float* init_param, void* workspace,
                              size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);

/* The backward of det_lookup_sparse, fused: per-unique-id gradients straight from the output gradient (ABI >= 8).
 * Inputs are the forward's ids int64[nnz], segment_ids int32[nnz] (ascending, in [0, batch)), weights f32[nnz] or NULL
 * and combiner, and gout f32[batch, dim] = dL/d(output).  The rule:
 *   den_b = the forward's normaliser of segment b, summed as the forward sums it: in id order from +0, the weights for
 *           DET_COMBINER_MEAN, sqrtf of the weights' squares for DET_COMBINER_SQRTN; none for DET_COMBINER_SUM;
 *   c_i   = w_i / den_{seg_i} (w_i = 1 without weights; c_i = w_i for DET_COMBINER_SUM), one IEEE division;
 *   g_i   = gout[seg_i, :] * c_i, one multiply per element;
 *   the gradient of a unique id (det_unique's first-occurrence order) = its g_i added in increasing position from 0.
 * den = 0 gives what IEEE division gives (inf / NaN), as in the forward.  The [nnz, dim] g_i are never materialised.
 * Malformed segment ids (not ascending, or outside [0, batch)) make every gradient NaN.
 * nnz == 0 is DET_OK (the count is 0); NULL ids, segment_ids or gout, a bad combiner, or batch == 0 with nnz > 0 are
 * DET_INVALID_ARGUMENT.
 *
 * det_lookup_sparse_grad: the backward alone, no table.  unique_out int64[nnz], grads_out f32[nnz, dim] (the first
 * *n_unique_dev rows are written), n_unique_dev: device int64.  Any dim.  workspace:
 * det_lookup_sparse_grad_workspace_bytes(nnz, batch, dim) bytes of device memory, 256 B aligned. */
size_t det_lookup_sparse_grad_workspace_bytes(size_t nnz, size_t batch, size_t dim);
det_status det_lookup_sparse_grad(const int64_t* ids, const int32_t* segment_ids, const float* weights, size_t nnz,
                                  size_t batch, int combiner, const float* gout, size_t dim, int64_t* unique_out,
                                  float* grads_out, int64_t* n_unique_dev, void* workspace, size_t workspace_bytes,
                                  det_stream_t stream);
/* det_apply_*_sparse: the backward above chained into the fused optimizer step of the matching det_apply_*_dup, in
 * one call with the unique count on the device (no host synchronisation).  Hyper-parameters, init_param (NULL on a
 * table with a keyed initializer), value dtypes, row limits, eviction scores and refusals: as det_apply_*_dup.
 * workspace: det_apply_sparse_workspace_bytes(nnz, batch, dim) bytes, 256 B aligned. */
size_t det_apply_sparse_workspace_bytes(size_t nnz, size_t batch, size_t dim);
det_status det_apply_adagrad_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                    size_t nnz, size_t batch, int combiner, const float* gout, float lr, float epsilon,
                                    const float* init_param, float init_accum, void* workspace, size_t workspace_bytes,
                                    int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_adam_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                 size_t nnz, size_t batch, int combiner, const float* gout, float alpha, float beta1,
                                 float beta2, float epsilon, const float* init_param, void* workspace,
                                 size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_sgd_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                size_t nnz, size_t batch, int combiner, const float* gout, float lr, float momentum,
                                int nesterov, const float* init_param, void* workspace, size_t workspace_bytes,
                                int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_ftrl_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                 size_t nnz, size_t batch, int combiner, const float* gout, float lr, float l1, float l2,
                                 float l2_shrinkage, const float* init_param, float init_accum, void* workspace,
                                 size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_rmsprop_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                    size_t nnz, size_t batch, int combiner, const float* gout, float lr, float rho,
                                    float momentum, float epsilon, int centered, int eps_in_sqrt,
                                    const float* init_param, float init_ms, void* workspace, size_t workspace_bytes,
                                    int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_adadelta_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                     size_t nnz, size_t batch, int combiner, const float* gout, float lr, float rho,
                                     float epsilon, const float* init_param, void* workspace, size_t workspace_bytes,
                                     int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_adamax_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                   size_t nnz, size_t batch, int combiner, const float* gout, float lr_t, float beta1,
                                   float beta2, float epsilon, const float* init_param, void* workspace,
                                   size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_nadam_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                  size_t nnz, size_t batch, int combiner, const float* gout, float lr, float beta1,
                                  float beta2, float epsilon, float omsn, float omsx, float omt, float mt1, float vden,
                                  const float* init_param, void* workspace, size_t workspace_bytes,
                                  int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_proximal_adagrad_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                             const float* weights, size_t nnz, size_t batch, int combiner,
                                             const float* gout, float lr, float l1, float l2, const float* init_param,
                                             float init_accum, void* workspace, size_t workspace_bytes,
                                             int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_proximal_sgd_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                         const float* weights, size_t nnz, size_t batch, int combiner, const float* gout,
                                         float lr, float l1, float l2, const float* init_param, void* workspace,
                                         size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_adagrad_da_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                       const float* weights, size_t nnz, size_t batch, int combiner, const float* gout,
                                       float lr, float l1, float l2, int64_t global_step, const float* init_param,
                                       float init_gg, void* workspace, size_t workspace_bytes,
                                       int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_adamw_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                  size_t nnz, size_t batch, int combiner, const float* gout, float alpha, float beta1,
                                  float beta2, float epsilon, float lr, float weight_decay, int amsgrad,
                                  const float* init_param, void* workspace, size_t workspace_bytes,
                                  int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_lion_sparse(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                 size_t nnz, size_t batch, int combiner, const float* gout, float lr, float beta1,
                                 float beta2, float weight_decay, const float* init_param, void* workspace,
                                 size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);

/* The backward of det_lookup_sparse_safe (ABI >= 8): the raw inputs of the forward, its combiner, has_default_id and
 * default_id, and gout f32[batch, dim].  The list is cleaned as the forward cleans it, except that with
 * has_default_id == 0 every empty row still gets its fill entry (id 0, weight 1): the reference looks id 0 up for
 * such rows and zeroes their output afterwards, so id 0 joins the unique set -- it is created and stepped -- with a
 * gradient contribution of exactly +0.0 from each such row, whatever gout holds there.  Every other gradient is
 * det_lookup_sparse_grad's rule on the cleaned list (positions of the cleaned list, first-occurrence order of its
 * ids).  Malformed segment ids give an empty cleaned list: no unique id, no step.  nnz == 0 is valid (every row is
 * empty); batch == 0 with nnz > 0 is DET_INVALID_ARGUMENT.
 *
 * det_lookup_sparse_safe_grad: the backward alone.  unique_out int64[nnz + batch], grads_out f32[nnz + batch, dim] (the
 * first *n_unique_dev rows are written).  workspace: det_lookup_sparse_safe_grad_workspace_bytes(nnz, batch, dim)
 * bytes, 256 B aligned. */
size_t det_lookup_sparse_safe_grad_workspace_bytes(size_t nnz, size_t batch, size_t dim);
det_status det_lookup_sparse_safe_grad(const int64_t* ids, const int32_t* segment_ids, const float* weights, size_t nnz,
                                       size_t batch, int combiner, int has_default_id, int64_t default_id,
                                       const float* gout, size_t dim, int64_t* unique_out, float* grads_out,
                                       int64_t* n_unique_dev, void* workspace, size_t workspace_bytes,
                                       det_stream_t stream);
/* det_apply_*_sparse_safe: that backward chained into the fused step of det_apply_*_sparse, in one call with every
 * count on the device.  The arguments are those of det_apply_*_sparse plus has_default_id and default_id; the
 * hyper-parameters, init_param, dtypes and refusals are the same (rows of dim % 4 == 0 and dim <= 128).
 * workspace: det_apply_sparse_safe_workspace_bytes(nnz, batch, dim) bytes, 256 B aligned. */
size_t det_apply_sparse_safe_workspace_bytes(size_t nnz, size_t batch, size_t dim);
det_status det_apply_adagrad_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                         const float* weights, size_t nnz, size_t batch, int combiner,
                                         int has_default_id, int64_t default_id, const float* gout, float lr,
                                         float epsilon, const float* init_param, float init_accum, void* workspace,
                                         size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_adam_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                      const float* weights, size_t nnz, size_t batch, int combiner, int has_default_id,
                                      int64_t default_id, const float* gout, float alpha, float beta1, float beta2,
                                      float epsilon, const float* init_param, void* workspace, size_t workspace_bytes,
                                      int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_sgd_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                     size_t nnz, size_t batch, int combiner, int has_default_id, int64_t default_id,
                                     const float* gout, float lr, float momentum, int nesterov, const float* init_param,
                                     void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                     det_stream_t stream);
det_status det_apply_ftrl_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                      const float* weights, size_t nnz, size_t batch, int combiner, int has_default_id,
                                      int64_t default_id, const float* gout, float lr, float l1, float l2,
                                      float l2_shrinkage, const float* init_param, float init_accum, void* workspace,
                                      size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_rmsprop_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                         const float* weights, size_t nnz, size_t batch, int combiner,
                                         int has_default_id, int64_t default_id, const float* gout, float lr, float rho,
                                         float momentum, float epsilon, int centered, int eps_in_sqrt,
                                         const float* init_param, float init_ms, void* workspace,
                                         size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_adadelta_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                          const float* weights, size_t nnz, size_t batch, int combiner,
                                          int has_default_id, int64_t default_id, const float* gout, float lr,
                                          float rho, float epsilon, const float* init_param, void* workspace,
                                          size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_adamax_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                        const float* weights, size_t nnz, size_t batch, int combiner,
                                        int has_default_id, int64_t default_id, const float* gout, float lr_t,
                                        float beta1, float beta2, float epsilon, const float* init_param,
                                        void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                        det_stream_t stream);
det_status det_apply_nadam_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                       const float* weights, size_t nnz, size_t batch, int combiner, int has_default_id,
                                       int64_t default_id, const float* gout, float lr, float beta1, float beta2,
                                       float epsilon, float omsn, float omsx, float omt, float mt1, float vden,
                                       const float* init_param, void* workspace, size_t workspace_bytes,
                                       int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_proximal_adagrad_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                                  const float* weights, size_t nnz, size_t batch, int combiner,
                                                  int has_default_id, int64_t default_id, const float* gout, float lr,
                                                  float l1, float l2, const float* init_param, float init_accum,
                                                  void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                                  det_stream_t stream);
det_status det_apply_proximal_sgd_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                              const float* weights, size_t nnz, size_t batch, int combiner,
                                              int has_default_id, int64_t default_id, const float* gout, float lr,
                                              float l1, float l2, const float* init_param, void* workspace,
                                              size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_adagrad_da_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                            const float* weights, size_t nnz, size_t batch, int combiner,
                                            int has_default_id, int64_t default_id, const float* gout, float lr,
                                            float l1, float l2, int64_t global_step, const float* init_param,
                                            float init_gg, void* workspace, size_t workspace_bytes,
                                            int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_adamw_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                       const float* weights, size_t nnz, size_t batch, int combiner, int has_default_id,
                                       int64_t default_id, const float* gout, float alpha, float beta1, float beta2,
                                       float epsilon, float lr, float weight_decay, int amsgrad,
                                       const float* init_param, void* workspace, size_t workspace_bytes,
                                       int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_lion_sparse_safe(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                      const float* weights, size_t nnz, size_t batch, int combiner, int has_default_id,
                                      int64_t default_id, const float* gout, float lr, float beta1, float beta2,
                                      float weight_decay, const float* init_param, void* workspace,
                                      size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);

/* det_apply_*_sparse_clip and det_apply_*_sparse_safe_clip: the steps of det_lookup_sparse_clip and
 * det_lookup_sparse_safe_clip (ABI >= 8).  The arguments are those of det_apply_*_sparse / det_apply_*_sparse_safe plus
 * max_norm after the combiner.  Each unique id's summed gradient G (det_lookup_sparse_grad's rule, unchanged) is taken
 * through the backward of the clip row -> row * c / max(||row||_2, c), c = max_norm, at the fp32 row p the step reads
 * (the stored row, or for a key the step creates its init_param / keyed initializer row: the row the clipped forward
 * read), then the optimizer rule runs on the result G':
 *   ss  = sum_k p_k * p_k, and dot = sum_k p_k * G_k, each reduced as det_lookup_sparse_clip reduces ||row||^2: every
 *         lane of a row group of lpr lanes (lpr = the power of two >= dim / 4) adds the products of its 4 elements in
 *         order, then an xor butterfly over the lpr lanes;
 *   !(sqrtf(ss) > c): G' = G bit for bit (the forward did not clip: its scale was exactly 1);
 *   otherwise:        s = c / sqrtf(ss), t = (s * dot) / ss, G'_k = G_k * s - p_k * t (J^T G, one fp32 rounding each).
 * The clip applies once per unique id, after the position-order sum, as the reference clips the unique rows before the
 * gather.  The step and the forward agree bit for bit on which rows were clipped when the forward ran its 16-byte
 * geometry: dim % 4 == 0 and `out` and `default_row` 16 B aligned (every cudaMalloc / torch allocation is).  With an
 * unaligned `out` or `default_row` the forward sums each row's squares one float per lane, in another order, so a row
 * whose norm is within rounding of max_norm may be clipped by one and not by the other.  max_norm == 0 is the unclipped call bit for bit; a negative or NaN max_norm is DET_INVALID_ARGUMENT;
 * max_norm > 0 on a DET_FLOAT16 / DET_BFLOAT16 table is DET_UNIMPLEMENTED (as det_lookup_sparse_clip).  Rows, eviction
 * scores, keyed initializers, slot dtypes and workspaces: as det_apply_*_sparse(_safe). */
det_status det_apply_adagrad_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                         const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                         const float* gout, float lr, float epsilon, const float* init_param,
                                         float init_accum, void* workspace, size_t workspace_bytes,
                                         int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_adam_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                      const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                      const float* gout, float alpha, float beta1, float beta2, float epsilon,
                                      const float* init_param, void* workspace, size_t workspace_bytes,
                                      int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_sgd_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids, const float* weights,
                                     size_t nnz, size_t batch, int combiner, float max_norm, const float* gout,
                                     float lr, float momentum, int nesterov, const float* init_param, void* workspace,
                                     size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_ftrl_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                      const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                      const float* gout, float lr, float l1, float l2, float l2_shrinkage,
                                      const float* init_param, float init_accum, void* workspace,
                                      size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_rmsprop_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                         const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                         const float* gout, float lr, float rho, float momentum, float epsilon,
                                         int centered, int eps_in_sqrt, const float* init_param, float init_ms,
                                         void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                         det_stream_t stream);
det_status det_apply_adadelta_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                          const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                          const float* gout, float lr, float rho, float epsilon,
                                          const float* init_param, void* workspace, size_t workspace_bytes,
                                          int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_adamax_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                        const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                        const float* gout, float lr_t, float beta1, float beta2, float epsilon,
                                        const float* init_param, void* workspace, size_t workspace_bytes,
                                        int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_nadam_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                       const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                       const float* gout, float lr, float beta1, float beta2, float epsilon, float omsn,
                                       float omsx, float omt, float mt1, float vden, const float* init_param,
                                       void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                       det_stream_t stream);
det_status det_apply_proximal_adagrad_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                                  const float* weights, size_t nnz, size_t batch, int combiner,
                                                  float max_norm, const float* gout, float lr, float l1, float l2,
                                                  const float* init_param, float init_accum, void* workspace,
                                                  size_t workspace_bytes, int64_t* n_unique_dev_out,
                                                  det_stream_t stream);
det_status det_apply_proximal_sgd_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                              const float* weights, size_t nnz, size_t batch, int combiner,
                                              float max_norm, const float* gout, float lr, float l1, float l2,
                                              const float* init_param, void* workspace, size_t workspace_bytes,
                                              int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_adagrad_da_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                            const float* weights, size_t nnz, size_t batch, int combiner,
                                            float max_norm, const float* gout, float lr, float l1, float l2,
                                            int64_t global_step, const float* init_param, float init_gg,
                                            void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                            det_stream_t stream);
det_status det_apply_adamw_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                       const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                       const float* gout, float alpha, float beta1, float beta2, float epsilon,
                                       float lr, float weight_decay, int amsgrad, const float* init_param,
                                       void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                       det_stream_t stream);
det_status det_apply_lion_sparse_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                      const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                      const float* gout, float lr, float beta1, float beta2, float weight_decay,
                                      const float* init_param, void* workspace, size_t workspace_bytes,
                                      int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_adagrad_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                              const float* weights, size_t nnz, size_t batch, int combiner,
                                              float max_norm, int has_default_id, int64_t default_id, const float* gout,
                                              float lr, float epsilon, const float* init_param, float init_accum,
                                              void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                              det_stream_t stream);
det_status det_apply_adam_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                           const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                           int has_default_id, int64_t default_id, const float* gout, float alpha,
                                           float beta1, float beta2, float epsilon, const float* init_param,
                                           void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                           det_stream_t stream);
det_status det_apply_sgd_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                          const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                          int has_default_id, int64_t default_id, const float* gout, float lr,
                                          float momentum, int nesterov, const float* init_param, void* workspace,
                                          size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_ftrl_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                           const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                           int has_default_id, int64_t default_id, const float* gout, float lr,
                                           float l1, float l2, float l2_shrinkage, const float* init_param,
                                           float init_accum, void* workspace, size_t workspace_bytes,
                                           int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_rmsprop_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                              const float* weights, size_t nnz, size_t batch, int combiner,
                                              float max_norm, int has_default_id, int64_t default_id, const float* gout,
                                              float lr, float rho, float momentum, float epsilon, int centered,
                                              int eps_in_sqrt, const float* init_param, float init_ms, void* workspace,
                                              size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_adadelta_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                               const float* weights, size_t nnz, size_t batch, int combiner,
                                               float max_norm, int has_default_id, int64_t default_id,
                                               const float* gout, float lr, float rho, float epsilon,
                                               const float* init_param, void* workspace, size_t workspace_bytes,
                                               int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_adamax_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                             const float* weights, size_t nnz, size_t batch, int combiner,
                                             float max_norm, int has_default_id, int64_t default_id, const float* gout,
                                             float lr_t, float beta1, float beta2, float epsilon,
                                             const float* init_param, void* workspace, size_t workspace_bytes,
                                             int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_nadam_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                            const float* weights, size_t nnz, size_t batch, int combiner,
                                            float max_norm, int has_default_id, int64_t default_id, const float* gout,
                                            float lr, float beta1, float beta2, float epsilon, float omsn, float omsx,
                                            float omt, float mt1, float vden, const float* init_param, void* workspace,
                                            size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_proximal_adagrad_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                                       const float* weights, size_t nnz, size_t batch, int combiner,
                                                       float max_norm, int has_default_id, int64_t default_id,
                                                       const float* gout, float lr, float l1, float l2,
                                                       const float* init_param, float init_accum, void* workspace,
                                                       size_t workspace_bytes, int64_t* n_unique_dev_out,
                                                       det_stream_t stream);
det_status det_apply_proximal_sgd_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                                   const float* weights, size_t nnz, size_t batch, int combiner,
                                                   float max_norm, int has_default_id, int64_t default_id,
                                                   const float* gout, float lr, float l1, float l2,
                                                   const float* init_param, void* workspace, size_t workspace_bytes,
                                                   int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_adagrad_da_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                                 const float* weights, size_t nnz, size_t batch, int combiner,
                                                 float max_norm, int has_default_id, int64_t default_id,
                                                 const float* gout, float lr, float l1, float l2, int64_t global_step,
                                                 const float* init_param, float init_gg, void* workspace,
                                                 size_t workspace_bytes, int64_t* n_unique_dev_out,
                                                 det_stream_t stream);
det_status det_apply_adamw_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                            const float* weights, size_t nnz, size_t batch, int combiner,
                                            float max_norm, int has_default_id, int64_t default_id, const float* gout,
                                            float alpha, float beta1, float beta2, float epsilon, float lr,
                                            float weight_decay, int amsgrad, const float* init_param, void* workspace,
                                            size_t workspace_bytes, int64_t* n_unique_dev_out, det_stream_t stream);
det_status det_apply_lion_sparse_safe_clip(det_table* t, const int64_t* ids, const int32_t* segment_ids,
                                           const float* weights, size_t nnz, size_t batch, int combiner, float max_norm,
                                           int has_default_id, int64_t default_id, const float* gout, float lr,
                                           float beta1, float beta2, float weight_decay, const float* init_param,
                                           void* workspace, size_t workspace_bytes, int64_t* n_unique_dev_out,
                                           det_stream_t stream);

/* ---- key-hash sharding across GPUs (python/ops/dynamic_embedding_variable.py:165-197 default_partition_fn,
 * python/ops/shadow_embedding_ops.py:397-447 alltoall exchange) ----
 * Partition n keys into num_shards contiguous groups by owner = (key & 0x7fffffff) % S (gpu_mode)
 * or floor-mod(key, S):  keys_out = keys grouped by owner (stable within a group),
 * perm_out[j] = original position of keys_out[j], counts_out[s] = keys owned by shard s (DEVICE int64[S]).
 * workspace: det_partition_workspace_bytes(n, S). */
size_t det_partition_workspace_bytes(size_t n, int num_shards);
det_status det_partition(const int64_t* keys, size_t n, int num_shards, int gpu_mode,
                         int64_t* keys_out, int32_t* perm_out, int64_t* counts_out, void* workspace,
                         size_t workspace_bytes, det_stream_t stream);
/* rows_out[perm[j],:] = rows_in[j,:]  (dynamic_stitch of the returned rows) and its inverse
 * rows_out[j,:] = rows_in[perm[j],:] (gather before sending values/grads to their owners). */
det_status det_scatter_rows(const void* rows_in, const int32_t* perm, size_t n, size_t row_bytes,
                            void* rows_out, det_stream_t stream);
det_status det_gather_rows(const void* rows_in, const int32_t* perm, size_t n, size_t row_bytes,
                           void* rows_out, det_stream_t stream);

/* ---- one table sharded over the GPUs of an NVSwitch box, accessed ONE-SIDED over NVLink peer memory
 * (replaces HvdVariable.__alltoall_embedding_lookup__, python/ops/shadow_embedding_ops.py:397-447: partition ->
 * alltoall(ids) -> local lookup -> alltoall(rows) -> scatter).  Every rank owns the shard owner(key) == rank,
 * exports CUDA-IPC handles of its planes (det_peer_export), gathers all ranks' handles (any transport) and
 * builds a group; det_peer_find / det_peer_insert then take keys owned by ANY rank: one kernel probes the owner's
 * key plane and moves the row over NVLink, no collective.  A published table cannot grow.
 * tables[p] non-NULL = shard p lives in this process (its own rank, or several shards faked on one GPU like the
 * reference's tests, kernel_tests/dynamic_embedding_ops_test.py:329); NULL = map it from handles[p].
 * det_peer_barrier: flag barrier over peer memory separating the "all ranks read" / "all ranks write" phases.
 * Shards with an eviction strategy (DET_FLAGS_EVICT) are served by their OWNERS only: the one-sided det_peer_find and
 * det_peer_insert return DET_INVALID_ARGUMENT for such a group.  Lookups go through det_peer_xchg_find; new keys enter
 * through det_peer_xchg_apply_* (find-or-insert inside the fused step: room by eviction, scores written by the kernel,
 * no host synchronisation below the load limit) or det_peer_xchg_insert (the owner compacts what arrived and runs its
 * own scored insert: ONE host synchronisation per call; DET_UNIMPLEMENTED for the CUSTOMIZED strategy, which needs
 * caller scores), or det_peer_route + inbox + the owner's own det_apply_* / det_insert_scored
 * (the reference: one HkvHashTable per Horovod rank behind HvdAllToAllEmbedding, keras/layers/embedding.py:545-595). */
typedef struct det_peer_group det_peer_group;
size_t det_peer_handle_bytes(void);
det_status det_peer_export(det_table* t, void* handle_out_host);
det_status det_peer_group_create(det_peer_group** out, det_table* const* tables, const void* handles_host,
                                 int world, int rank, int gpu_mode);
det_status det_peer_group_destroy(det_peer_group* g);
/* Same group over SYMMETRIC-MEMORY regions (preferred: CUDA VMM mappings keep 2 MB pages; legacy CUDA-IPC imports
 * make random access over a 50 GB shard TLB-bound).  Every rank builds its shard with det_table_create_in_region
 * in a region all peers have mapped; region_ptrs[p] = where THIS process sees rank p's region. */
det_status det_peer_group_create_regions(det_peer_group** out, det_table* local, const void* const* region_ptrs,
                                         int world, int rank, int gpu_mode);
det_status det_peer_find(det_peer_group* g, const int64_t* keys, size_t n, const void* defaults,
                         int full_size_default, void* values_out, uint8_t* exists, det_stream_t stream);
det_status det_peer_insert(det_peer_group* g, const int64_t* keys, const void* values, size_t n,
                           det_stream_t stream);
det_status det_peer_barrier(det_peer_group* g, det_stream_t stream);
/* One-sided all-to-all-v of (key, row) pairs -- hvd.alltoall(ids, splits) + hvd.alltoall(rows, splits)
 * (python/ops/shadow_embedding_ops.py:420-441) as ONE kernel: det_peer_route partitions the batch by owner and writes
 * every pair into its segment of the owner's peer-mapped INBOX with posted NVLink stores, then publishes the counts.
 * After det_peer_barrier the owner reads how much every source sent (det_peer_inbox_counts, HOST out, syncs) and
 * concatenates the segments (det_peer_inbox_gather).  Backward path: row gradients travel to the owner, which
 * combines duplicates and runs the fused optimizer locally (half-sync, dynamic_embedding_optimizer.py:580-595).
 * inbox_ptrs[p] = where THIS process sees rank p's inbox (det_peer_inbox_bytes each, zeroed by its owner). */
size_t det_peer_inbox_bytes(int world, size_t max_items, size_t row_bytes);
det_status det_peer_inbox_attach(det_peer_group* g, const void* const* inbox_ptrs, size_t max_items, size_t row_bytes);
det_status det_peer_route(det_peer_group* g, const int64_t* keys, const void* rows, size_t n, det_stream_t stream);
det_status det_peer_inbox_counts(det_peer_group* g, int shard, int64_t* counts_host, det_stream_t stream);
det_status det_peer_inbox_gather(det_peer_group* g, int shard, const int64_t* counts_host, int64_t* keys_out,
                                 void* rows_out, det_stream_t stream);

/* ---- owner-side exchange: the sharded Find / Insert with PUSHES only (ABI >= 5) ----
 * Replaces HvdVariable.__alltoall_embedding_lookup__ (python/ops/shadow_embedding_ops.py:397-447: alltoall(ids) ->
 * local lookup -> alltoall(rows) -> scatter) and the reverse path of the write-back, without a collective library and
 * without the remote probe reads of det_peer_find / det_peer_insert: ids travel to the owner's MAILBOX with posted
 * NVLink stores, the owner probes its own shard at HBM speed and stores every row straight into the requester's
 * output ring at the id's position; inserts travel as (key, row) pairs and are applied by the owner locally.
 * Ordering: per-(source, owner) flag words in the mailbox (st.release.sys / ld.acquire.sys), no rank-wide barrier.
 * COLLECTIVE: every rank of the group issues the same sequence of det_peer_xchg_find / det_peer_xchg_insert calls on ONE
 * stream per group (n may differ per rank, 0 allowed) -- the contract of the reference's alltoall ops.
 * mailbox_ptrs[p] = where THIS process sees rank p's mailbox (det_peer_xchg_bytes each, zeroed by its owner before
 * any rank attaches; ranks synchronise on the host between zeroing and the first call).  max_items bounds one call's n.
 * det_peer_xchg_find: rows land in this rank's 2-entry output ring; *rows_view (nullable) = device pointer of the n
 * rows, valid until the next-but-one det_peer_xchg_find; values_out (nullable) receives a copy; exists_out nullable.
 * With full_size_default = 0 the broadcast default row must be identical on every rank (the owner writes it).
 * A full shard is reported by DET_TABLE_FULL of a LATER call (asynchronous state snapshots), never silently. */
size_t det_peer_xchg_bytes(int world, size_t max_items, size_t row_bytes);
det_status det_peer_xchg_attach(det_peer_group* g, const void* const* mailbox_ptrs, size_t max_items, size_t row_bytes);
det_status det_peer_xchg_find(det_peer_group* g, const int64_t* keys, size_t n, const void* defaults,
                              int full_size_default, void* values_out, uint8_t* exists_out, void** rows_view,
                              det_stream_t stream);
det_status det_peer_xchg_insert(det_peer_group* g, const int64_t* keys, const void* values, size_t n,
                                det_stream_t stream);

/* Sharded sparse optimizer step through the owners (ABI >= 7): the backward of the sharded lookup -- the gradient of
 * HvdVariable.__alltoall_embedding_lookup__ followed by the optimizer patch (python/ops/shadow_embedding_ops.py:397-447,
 * python/ops/dynamic_embedding_optimizer.py:150-204; half-sync: sparse rows are never all-reduced, :580-595).
 * COLLECTIVE like det_peer_xchg_insert.  Every rank routes its (unique id, row gradient) pairs to the owners; the owner
 * compacts what arrived, sums the gradients several ranks sent for one id (position order: source rank, then the
 * sender's order) and runs the fused find-or-insert optimizer step on its shard (det_apply_*_dup on the device-side
 * count).  No cudaStreamSynchronize and no host round trip for split sizes (the reference negotiates them on the host,
 * shadow_embedding_ops.py:414-421).  workspace: det_peer_xchg_apply_workspace_bytes(g) bytes, 256 B aligned. */
size_t det_peer_xchg_apply_workspace_bytes(det_peer_group* g);
det_status det_peer_xchg_apply_adagrad(det_peer_group* g, const int64_t* keys, const float* grads, size_t n, float lr,
                                       float epsilon, const float* init_param, float init_accum, void* workspace,
                                       size_t workspace_bytes, det_stream_t stream);
det_status det_peer_xchg_apply_adam(det_peer_group* g, const int64_t* keys, const float* grads, size_t n, float alpha,
                                    float beta1, float beta2, float epsilon, const float* init_param, void* workspace,
                                    size_t workspace_bytes, det_stream_t stream);

/* ---- file-system format of SaveToFileSystem / LoadFromFileSystem
 * (cuckoo_hashtable_op.cc:310-504): raw little-endian `<prefix>-keys` (int64[n]) and
 * `<prefix>-values` (V[n*dim]).  HOST paths; synchronous. ---- */
/* attrs of the ops: buffer_size (keys per chunk; memory use is bounded by it), append_to_file, and -- for
 * load_entire_dir (cuckoo_hashtable_op.cc:477-498) -- clear_first = 0 to add one more `<name>_mht_*` file to a table
 * that was cleared by the first call. */
det_status det_save(det_table* t, const char* prefix, size_t buffer_keys, int append_to_file);
det_status det_load(det_table* t, const char* prefix, size_t buffer_keys, int clear_first);

/* Checkpointing the state of the FUSED optimizers.  The reference keeps every optimizer slot in its own table
 * `<var>/<opt>/<slot>` (python/ops/dynamic_embedding_optimizer.py:870-958), saved and restored like any variable;
 * here the slots are planes of the variable's own table, so they travel as one more raw file pair per plane:
 *   det_save_plane  = det_save of plane 1..num_slot_planes (rows in the plane's dtype: fp32, or the table's fp16 / bf16
 *                     with DET_FLAGS_SLOTS_IN_VALUE_DTYPE -- the reference's slot files of a half variable; never-stepped
 *                     keys carry the slot initializer),
 *   det_load_plane  = the pair read back into the plane for the keys that are IN the table (restore the value plane
 *                     first); keys of the file that are not in the table are skipped.  The `-values` file of an fp16 /
 *                     bf16 plane must hold exactly n * dim * 2 bytes for the n keys of `-keys` (an fp32 file is refused
 *                     with DET_IO_ERROR, not misread),
 *   det_import_plane = the same from device buffers (keys int64 [n], rows fp32 [n, dim]), asynchronous on `stream`; rows
 *                     are rounded to nearest even into an fp16 / bf16 plane (exact for rows widened from that dtype).
 * ABI >= 4. */
det_status det_import_plane(det_table* t, int plane, const int64_t* keys, const float* rows, size_t n,
                            det_stream_t stream);
det_status det_save_plane(det_table* t, int plane, const char* prefix, size_t buffer_keys, int append_to_file);
det_status det_load_plane(det_table* t, int plane, const char* prefix, size_t buffer_keys);

/* introspection for tests / benches (HOST outs; synchronises) */
typedef struct det_stats {
  int64_t size;        /* live keys */
  int64_t used_slots;  /* non-empty slots (live + tombstones) */
  uint64_t capacity;   /* slots */
  uint64_t buckets;
  uint64_t hbm_bytes;  /* device bytes held by the table (slot planes at their element size) */
  uint32_t error_flags;
  uint32_t rehash_count;
  uint32_t evict_events;  /* eviction events so far (ABI >= 2) */
  uint32_t reserved;
  uint64_t evicted_keys;  /* keys evicted so far */
  uint64_t host_bytes;    /* ABI >= 3: bytes of the value plane that live in host memory (max_hbm_for_vectors);
                           * hbm_bytes excludes them */
} det_stats;
det_status det_get_stats(det_table* t, det_stats* out_host, det_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* DETABLE_H_ */
