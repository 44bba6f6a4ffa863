/*
 * er_b200.h -- C ABI of liber_b200.so: the sm_90a kernels behind EasyRec's
 * sparse-embedding + feature-interaction training path.
 *
 * The reference (alibaba/EasyRec) has NO native ABI on this path: the path is a
 * TensorFlow graph assembled in Python (SURVEY.md section 8b).  Every entry
 * point below therefore cites the reference *Python* call it replaces; the
 * ctypes binding a maintainer would add is shown in INTEGRATION.md.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller unless the
 *     parameter is documented "host"; nothing here allocates or frees device
 *     memory, and there is no hidden global state;
 *   - every call enqueues work on `stream` (a cudaStream_t passed as void*) and
 *     returns immediately; it is CUDA-graph capturable;
 *   - return value: 0 = ER_OK, anything else is an er_status; the message for
 *     the calling thread's last failure is er_last_error();
 *   - "rows" are int64 row numbers inside one embedding ARENA (all tables with
 *     the same embedding_dim packed back to back); -1 marks a dropped lookup;
 *   - segments are the (slot, sample) cells of the reference's packed CSR
 *     layout (feature-major, easy_rec/python/input/load_parquet.py:81-90).
 */
#ifndef ER_B200_H_
#define ER_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ER_B200_ABI_VERSION 3

typedef void* er_stream_t; /* cudaStream_t */

typedef enum er_status {
  ER_OK = 0,
  ER_ERR_INVALID_ARG = 1,
  ER_ERR_WORKSPACE = 2,
  ER_ERR_CUDA = 3,
  ER_ERR_UNSUPPORTED = 4
} er_status;

/* raw value -> table row rule (SURVEY.md A.1) */
typedef enum er_bucket_mode {
  /* row = Fingerprint64(as_string(v)) mod hash_bucket_size
   * (feature_column_v2.py:3915-3921, input/input.py:356-376,541-543) */
  ER_BUCKET_FARM_DECIMAL = 0,
  /* row = v floormod num_buckets (input/parquet_input.py:221) */
  ER_BUCKET_MOD = 1,
  /* v == -1 dropped (feature_column_v2.py:2566-2585); v < 0 or v >= num_buckets
   * -> default 0 (feature_column_v2.py:4268-4292, feature_column.py:293-294) */
  ER_BUCKET_IDENTITY = 2,
  /* already a table-local row (e.g. RawFeature projection ids 0..k-1,
   * input/input.py:648-673); v < 0 dropped */
  ER_BUCKET_NONE = 3,
  /* the slot's table has exactly ONE row (RawFeature projection with raw_input_dim 1,
   * input/input.py:648-673: id 0 weighted by the value) and no other slot of the call reads it:
   * every value >= 0 maps to that row, < 0 is dropped.  er_embedding_bwd does not send these lookups
   * through the dedup: the row's gradient is the weighted column sum of the slot's gradient block. */
  ER_BUCKET_ONE_ROW = 4,
  /* vocabulary column (categorical_column_with_vocabulary_{list,file} with default_value 0 and no OOV buckets,
   * feature_column/feature_column.py:277-290,320-333,497-509): v is the 63-bit key of the raw string
   * (Fingerprint64(bytes) % (2^63 - 1)); row = the position of the vocabulary entry with key v, 0 when no entry
   * has it; v < 0 dropped.  num_buckets = the vocabulary's size.  The entries live in a read-only index
   * (er_vocab_t) that only the *_vocab forms of K1 are given. */
  ER_BUCKET_VOCAB = 5
} er_bucket_mode;

/* safe_embedding_lookup_sparse combiners (compat/embedding_ops.py:37-162,
 * compat/feature_column/feature_column.py:202-244) */
typedef enum er_combiner {
  ER_COMBINER_SUM = 0,
  ER_COMBINER_MEAN = 1,
  ER_COMBINER_SQRTN = 2,
  /* flag, OR-ed into er_slot_t.combiner: every entry of weights[] that belongs to this slot is 1.0 (single-valued id
   * slots of a call whose weights array exists only for other slots); the backward then skips the per-lookup read */
  ER_COMBINER_UNIT_WEIGHTS = 16
} er_combiner;

/* One embedding slot = one (feature column, output position) pair; the
 * host-side table plan (FeatureColumnParser equivalent) fills an array of
 * these once and uploads it. 48 bytes, no pointers. */
typedef struct er_slot {
  int64_t num_buckets; /* hash_bucket_size | num_buckets of the column        */
  int64_t row_offset;  /* first arena row of the column's table               */
  int32_t seg_begin;   /* first segment (global numbering) of this slot       */
  int32_t n_seg;       /* segments of this slot: B, or B*T for sequence slots */
  int32_t bucket_mode; /* er_bucket_mode                                      */
  int32_t combiner;    /* er_combiner                                         */
  int32_t out_buf;     /* index into the out_bufs[] / grad_bufs[] argument    */
  int32_t out_stride;  /* row stride of that buffer, in floats                */
  int32_t out_col;     /* first column of this slot inside a buffer row       */
  int32_t shard_n;     /* >1: rows are mod-sharded over shard_n ranks
                          (feature_column.py:296,317,461-463)                 */
} er_slot_t;

#define ER_MAX_BUFS 8

typedef enum er_opt_kind {
  ER_OPT_SGD = 0,
  ER_OPT_ADAGRAD = 1,   /* tf.train.AdagradOptimizer sparse apply            */
  ER_OPT_LAZY_ADAM = 2, /* compat/adam_s.py:185-213                          */
  ER_OPT_ADAM_ROWS = 3, /* tf.train.AdamOptimizer (builders/optimizer_builder.py:61-66):
                           touched rows take the same row rule as lazy Adam in
                           er_embedding_bwd; every other row decays in
                           er_adam_dense_sweep (behaviour documented at
                           compat/adam_s.py:74-81)                            */
  ER_OPT_MOMENTUM = 4   /* tf.train.MomentumOptimizer (builders/optimizer_builder.py:91-97,
                           momentum_optimizer_value > 0): accum = accum * momentum + g,
                           var -= lr * accum on the touched rows (SparseApplyMomentum);
                           one state array (accum, starts at 0); momentum travels in
                           er_opt_t.beta1                                        */
} er_opt_kind;

/* Step-varying hyper-parameters in DEVICE memory (er_opt_t.hyper_dev): the kernels read them at run
 * time, so one captured CUDA graph follows a learning-rate schedule and Adam's beta powers. */
enum {
  ER_HYPER_LR = 0,          /* learning rate of this step (core/learning_schedules.py:30-75) */
  ER_HYPER_BETA1_POWER = 1, /* beta1^t before this step's _finish (compat/adam_s.py:233-245) */
  ER_HYPER_BETA2_POWER = 2,
  ER_HYPER_GRAD_SCALE = 3,
  ER_HYPER_N = 4
};

typedef struct er_opt {
  int32_t kind;      /* er_opt_kind */
  float lr;          /* learning rate of this step (host-side schedule)       */
  float beta1;
  float beta2;
  float eps;
  float beta1_power; /* beta1^t BEFORE this step's _finish (adam_s.py:233-245) */
  float beta2_power;
  float grad_scale;  /* multiplies the summed gradient: 1/N for sharded tables
                        (compat/optimizers.py:315-316) times
                        embedding_learning_rate_multiplier
                        (model/easy_rec_estimator.py:308-317)                 */
  const float* hyper_dev; /* NULL, or DEVICE float[ER_HYPER_N] that overrides lr,
                             beta1_power, beta2_power and grad_scale above      */
} er_opt_t;

/* ---- library ---------------------------------------------------------- */
int er_abi_version(void);
const char* er_last_error(void);
/* kernels this library has enqueued since load (bench.py's gpu_launches) */
uint64_t er_launch_count(void);

/* ---- K0: lens -> CSR --------------------------------------------------
 * row_ptr[0]=0, row_ptr[s+1]=row_ptr[s]+lens[s]; seg_ids[l]=s for the lookups
 * of segment s.  Replaces cumsum(segment_lens) + searchsorted
 * (compat/feature_column/feature_column.py:264-266).
 * ws: er_csr_workspace_bytes(n_seg) bytes. */
size_t er_csr_workspace_bytes(int64_t n_seg);
int er_csr_from_lens(const int32_t* lens, int64_t n_seg, int32_t* row_ptr,
                     int32_t* seg_ids, int64_t n_lookups_cap, void* ws,
                     size_t ws_bytes, er_stream_t stream);

/* ---- K1: raw ids -> arena rows ---------------------------------------
 * rows[l] = slot.row_offset + bucket(ids[l]) per the slot's er_bucket_mode,
 * or -1 when the lookup is dropped.  With shard_n > 1 the result is the
 * owner-local row and owner[l] (may be NULL) receives id mod shard_n
 * (-1 for a dropped lookup).
 * seg_ids == NULL means lookup l belongs to segment l (single-valued slots);
 * row_ptr == NULL means exactly n_lookups_cap lookups, else row_ptr[n_seg]. */
int er_bucketize(const int64_t* ids, const int32_t* seg_ids,
                 const int32_t* row_ptr, int64_t n_seg, int64_t n_lookups_cap,
                 const er_slot_t* slots, int32_t n_slots, int64_t* rows,
                 int32_t* owner, er_stream_t stream);
/* er_bucketize given the lookup weights that K2 and K7 will be given (NULL:
 * the same as er_bucketize).  A lookup of a mean / sqrtn slot whose weight is
 * not > 0 (NaN included) is dropped here (safe_embedding_lookup_sparse's
 * _prune_invalid_weights, compat/embedding_ops.py), so that K2, K7,
 * er_mark_rows and K8 agree that its row is not looked up; sum slots keep
 * every weight.  Weighted calls with mean / sqrtn slots must use this form. */
int er_bucketize_weighted(const int64_t* ids, const float* weights, const int32_t* seg_ids,
                          const int32_t* row_ptr, int64_t n_seg, int64_t n_lookups_cap,
                          const er_slot_t* slots, int32_t n_slots, int64_t* rows,
                          int32_t* owner, er_stream_t stream);

/* er_bucketize over un-pooled histories (SequenceFeature slots without a
 * combiner): ids and rows are [n_features, batch, seq_len] steps, step
 * l = (f*batch + b)*seq_len + t is segment l of the slot plan, and
 * lens[f*batch + b] is the length of that sample's history.  A step with
 * t >= lens[...] is padding: rows[l] = owner[l] = -1 and its id is not read,
 * so K8 never requests it.  A length below 0 pads every step and one above
 * seq_len pads none (lengths are clamped to [0, seq_len]).  Live steps follow
 * er_bucketize bit for bit (rows, owner and dropped ids).  One launch,
 * deterministic, no allocation; n_features*batch*seq_len < 2^31. */
int er_bucketize_seq(const int64_t* ids, const int32_t* lens, int64_t batch,
                     int32_t seq_len, int32_t n_features, const er_slot_t* slots,
                     int32_t n_slots, int64_t* rows, int32_t* owner,
                     er_stream_t stream);

/* A vocabulary's index for ER_BUCKET_VOCAB slots: the layout of a key-value table's index (ER_KV_EMPTY = free
 * entry, n_index a power of two >= 16), built once with er_kv_insert_rows from the entries' keys and their
 * positions, and never written after.  DEVICE memory, like the arrays it points to. */
typedef struct er_vocab {
  const int64_t* index_keys;
  const int64_t* index_rows;
  int64_t n_index;
} er_vocab_t;

/* er_bucketize_weighted for slot plans with ER_BUCKET_VOCAB slots: vocabs (DEVICE, n_slots entries) holds slot i's
 * vocabulary at vocabs[i] (the entries of other slots are not read).  A hit reads the entry's position, a miss
 * row 0, a key < 0 is dropped; then row_offset, shard_n and the weight pruning apply as for every other mode.  Every
 * other slot gives er_bucketize_weighted's result bit for bit.  One launch. */
int er_bucketize_vocab(const int64_t* ids, const float* weights, const int32_t* seg_ids,
                       const int32_t* row_ptr, int64_t n_seg, int64_t n_lookups_cap,
                       const er_slot_t* slots, int32_t n_slots, const er_vocab_t* vocabs,
                       int64_t* rows, int32_t* owner, er_stream_t stream);
/* er_bucketize_seq with vocabularies, as er_bucketize_vocab; padded steps are -1 and their ids are not read. */
int er_bucketize_seq_vocab(const int64_t* ids, const int32_t* lens, int64_t batch,
                           int32_t seq_len, int32_t n_features, const er_slot_t* slots,
                           int32_t n_slots, const er_vocab_t* vocabs, int64_t* rows,
                           int32_t* owner, er_stream_t stream);

/* ---- K8: index bucketing of the row-sharded lookup --------------------
 * Replaces the Unique + dynamic_partition + host-read split sizes of
 * embedding_parallel_lookup (compat/feature_column/feature_column.py:258-303).
 * rows / owner: er_bucketize's outputs under shard_n = world.  Distinct
 * (owner, row) pairs are grouped by owner into FIXED-capacity blocks, so the
 * all-to-alls that follow use equal splits and need no host round trip:
 *   send_rows[o*cap_per_peer + k] = k-th distinct row owned by rank o, -1 padding
 *   pos[l]    = o*cap_per_peer + k for lookup l (-1: dropped lookup)
 *   counts[o] = distinct rows owned by o; counts[world] = lookups lost because a
 *               block overflowed (the caller must treat > 0 as an error)
 * The k a row receives is not deterministic; no sum depends on it (see
 * csrc/shard_group.cu).  ws: er_shard_group_workspace_bytes(n_lookups). */
size_t er_shard_group_workspace_bytes(int64_t n_lookups);
int er_shard_group(const int64_t* rows, const int32_t* owner, int64_t n_lookups,
                   int32_t world, int64_t cap_per_peer, int64_t* send_rows,
                   int64_t* pos, int32_t* counts, void* ws, size_t ws_bytes,
                   er_stream_t stream);

/* Scalar helpers used by tests and by host-side plan code (host pointers). */
uint64_t er_fingerprint64_host(const char* s, size_t len);

/* ---- K2: multi-slot gather + pool ------------------------------------
 * For every segment s of every slot: out = combine_l w_l * table[rows[l]]
 * with safe_embedding_lookup_sparse pruning (rows<0 dropped; w<=0 dropped
 * unless combiner is sum; empty -> zeros).  Writes
 *   out_bufs[slot.out_buf][(s-slot.seg_begin)*out_stride + out_col + 0..dim)
 * i.e. the per-group concat of feature_column.input_layer
 * (compat/feature_column/feature_column.py:384-414) is fused into the store.
 * Inside a segment the terms w_l * row are added in lookup order, with
 * separate multiply and add (no FMA contraction).
 * seg_scale (n_seg floats, may be NULL when every slot is sum) receives the
 * mean/sqrtn denominators' reciprocal for the backward pass: 1/sum w for mean,
 * 1/sqrt(sum w^2) for sqrtn, 0 for an empty (or wholly pruned) mean / sqrtn
 * segment, and exactly 1 for every segment of a sum slot, empty ones included.
 * Lookups past min(n_lookups_cap, row_ptr[n_seg]) are not read.
 * At dim 4, 8, 16, 32, 64 and 128 (when table, row_stride and every out_bufs
 * base are 16-byte aligned) rows are moved with 16-byte accesses at
 * out_bufs[out_buf] + s*out_stride + out_col, and er_embedding_bwd reads
 * grad_bufs the same way: every slot's out_stride and out_col must then be
 * multiples of 4.  The slot table is device memory, so the kernels cannot
 * check this; the host-side plan builders refuse plans that break it.
 * out_bufs is a HOST array of n_bufs (<= ER_MAX_BUFS) device pointers. */
int er_embedding_fwd(const float* table, int64_t n_rows, int32_t dim,
                     int32_t row_stride, const int64_t* rows,
                     const float* weights, const int32_t* row_ptr,
                     int64_t n_seg, int64_t n_lookups_cap,
                     const er_slot_t* slots, int32_t n_slots,
                     float* const* out_bufs, int32_t n_bufs, float* seg_scale,
                     er_stream_t stream);

/* ---- K7: backward = dedup + segment-sum + fused optimizer row update ---
 * The IndexedSlices gradient of K2 (one row per lookup:
 * coef_l * grad_bufs[..][segment of l]) is summed per distinct row in
 * ascending lookup order (the lookups are hashed into buckets by row and each
 * bucket is sorted on (row, lookup) in shared memory: the deterministic
 * equivalent of TF's _deduplicate_indexed_slices), multiplied by
 * opt.grad_scale, and applied to the row and its optimizer state in the
 * same kernel.  Rows with many lookups are summed by a fixed chunked tree
 * instead (deterministic, but not the sequential order): runs of more than
 * 64 lookups when uniq_rows is given, otherwise runs of more than 48 in a
 * bucket that a whole CTA sorts.  When uniq_rows is given and dim is 1 or a
 * vector width up to 32, shorter runs are also summed by a fixed tree (a
 * warp's shuffle scan).  Slots of mode ER_BUCKET_ONE_ROW take a weighted
 * column sum instead.  Every lookup with rows[l] >= 0 counts as touching its
 * row (even with a zero coefficient), so rows must already carry -1 for the
 * lookups safe_embedding_lookup_sparse prunes: er_bucketize_weighted given
 * the same weights does that.  state0/state1: adagrad accumulator | adam m, v (same
 * layout and stride as table; unused ones NULL).  dim is at most 4096.
 * Rows, state and gradient buffers that are not 16-byte aligned (or a
 * row_stride that is not a multiple of 4) take a scalar path with the same
 * result as the aligned call wherever both sum in lookup order.
 * When uniq_rows/uniq_grads are non-NULL the deduplicated gradient is ALSO
 * written there (compact, sorted by row; *n_uniq receives the count); pass
 * table == NULL to only emit it. */
size_t er_embedding_bwd_workspace_bytes(int64_t n_lookups_cap, int32_t dim);
int er_embedding_bwd(float* table, float* state0, float* state1,
                     int64_t n_rows, int32_t dim, int32_t row_stride,
                     const int64_t* rows, const float* weights,
                     const int32_t* seg_ids, const int32_t* row_ptr,
                     int64_t n_seg, int64_t n_lookups_cap,
                     const er_slot_t* slots, int32_t n_slots,
                     const float* const* grad_bufs, int32_t n_bufs,
                     const float* seg_scale, const er_opt_t* opt,
                     int64_t* uniq_rows, float* uniq_grads, int32_t* n_uniq,
                     void* ws, size_t ws_bytes, er_stream_t stream);

/* The row-only half of er_embedding_bwd's dedup (hashing the lookups into buckets): it depends only on the
 * looked-up rows, not on any gradient, so it can run as soon as er_bucketize has produced them (e.g. on a side
 * stream under the dense forward/backward).  Takes the same rows / seg_ids / row_ptr / slots as the
 * er_embedding_bwd it prepares.  Leaves its result in `ws`; finish with
 * er_embedding_bwd_reuse_sort(..., sorted_ws = ws, sorted_dim = dim). */
int er_embedding_bwd_presort(const int64_t* rows, int64_t n_rows, const int32_t* seg_ids,
                             const int32_t* row_ptr, int64_t n_seg, int64_t n_lookups_cap,
                             const er_slot_t* slots, int32_t n_slots, int32_t dim, void* ws,
                             size_t ws_bytes, er_stream_t stream);

/* Same as er_embedding_bwd when the SAME rows array (same n_rows, same slot rules - e.g. the wide dim-1 table
 * next to the deep table of DeepFM / Wide&Deep) was already prepared by er_embedding_bwd_presort or
 * deduplicated by an earlier er_embedding_bwd on this stream whose workspace is sorted_ws (allocated for
 * dimension sorted_dim and left untouched since): only the per-row sums and the row updates run.  `ws` is this
 * call's own workspace (er_embedding_bwd_workspace_bytes(n, dim)).  uniq_rows output is not available here.
 * Precondition: dim and sorted_dim are in the same placement mode - both in {1, 4, 8, 16, 32} (warp-sized buckets)
 * or both outside it (CTA-sized buckets).  The reused placement is then the one this call would have made, so the
 * result equals er_embedding_bwd's bit for bit.  A placement of the other mode returns ER_ERR_UNSUPPORTED before
 * anything is written. */
int er_embedding_bwd_reuse_sort(float* table, float* state0, float* state1, int64_t n_rows,
                                int32_t dim, int32_t row_stride, const int64_t* rows,
                                const float* weights, const int32_t* seg_ids,
                                const int32_t* row_ptr, int64_t n_seg, int64_t n_lookups_cap,
                                const er_slot_t* slots, int32_t n_slots,
                                const float* const* grad_bufs, int32_t n_bufs,
                                const float* seg_scale, const er_opt_t* opt, int64_t* uniq_rows,
                                float* uniq_grads, int32_t* n_uniq, void* ws, size_t ws_bytes,
                                const void* sorted_ws, size_t sorted_ws_bytes, int32_t sorted_dim,
                                er_stream_t stream);

/* Apply an already deduplicated sparse gradient (rows distinct). */
int er_sparse_apply(float* table, float* state0, float* state1, int32_t dim,
                    int32_t row_stride, const int64_t* uniq_rows,
                    const float* uniq_grads, const int32_t* n_uniq,
                    int64_t n_cap, const er_opt_t* opt, er_stream_t stream);

/* TF AdamOptimizer's dense part for rows NOT touched this step
 * (documented at compat/adam_s.py:74-81): m*=b1, v*=b2, w-=lr_t*m/(sqrt(v)+eps)
 * streamed over the whole table; touched[] (n_rows bytes) masks rows already
 * updated by er_embedding_bwd.  Rows whose m and v are both zero are left unwritten
 * (their update is exactly zero), so a mostly-cold table costs one read pass. */
int er_adam_dense_sweep(float* table, float* m, float* v, int64_t n_rows,
                        int32_t dim, int32_t row_stride,
                        const uint8_t* touched, const er_opt_t* opt,
                        er_stream_t stream);

/* touched[rows[l]] = value for every live lookup (mask for er_adam_dense_sweep). */
int er_mark_rows(const int64_t* rows, int64_t n_lookups_cap, const int32_t* n_dev,
                 int64_t n_rows, uint8_t* touched, int32_t value,
                 er_stream_t stream);

/* ---- stable radix sort / unique (exposed for the sharded path) -------- */
size_t er_sort_workspace_bytes(int64_t n);
/* keys_out sorted ascending, vals_out = original positions (stable). */
int er_sort_rows(const int64_t* rows, int64_t n, const int32_t* n_dev,
                 int64_t max_row, uint32_t* keys_out, uint32_t* vals_out,
                 void* ws, size_t ws_bytes, er_stream_t stream);

/* ---- K3: FM second order ----------------------------------------------
 * y[b,:] = 0.5*((sum_f x[b,f,:])^2 - sum_f x[b,f,:]^2)   (layers/fm.py:20-26)
 * x is [B, F*D] with row stride x_stride. */
int er_fm_fwd(const float* x, int64_t batch, int32_t n_field, int32_t dim,
              int32_t x_stride, float* y, er_stream_t stream);
/* gx[b,f,:] (+)= gy[b,:] * (sum_f' x[b,f',:] - x[b,f,:]) */
int er_fm_bwd(const float* x, const float* gy, int64_t batch, int32_t n_field,
              int32_t dim, int32_t x_stride, float* gx, int32_t gx_stride,
              int32_t accumulate, er_stream_t stream);

/* FM block of DeepFM in one pass per direction (one warp per sample row, the row stays in registers):
 *   fwd: y as er_fm_fwd; *sumsq_out = sum_{b,f,d} x^2 - the embedding-regulariser term
 *        0.5*scale*||e||^2 of layers/input_layer.py:369-375 (NULL: skipped).  Deterministic.
 *   bwd: gx = g_pass + gy*(sum_f x - x) + (*coef_dev * coef_mul)*x  - the gradients of the deep tower
 *        input (g_pass, NULL = 0), of FM (gy, NULL = 0) and of the regulariser (coef_dev device scalar,
 *        NULL = 0) that all land on the same group matrix.
 * dim = 4*2^k <= 128, n_field*dim <= 1024, rows 16-byte aligned.  ws (er_fm_block_workspace_bytes)
 * must be zero-filled once by the caller; the kernel leaves it reusable. */
size_t er_fm_block_workspace_bytes(int64_t batch);
int er_fm_block_fwd(const float* x, int64_t batch, int32_t n_field, int32_t dim, int32_t x_stride,
                    float* y, float* sumsq_out, void* ws, size_t ws_bytes, er_stream_t stream);
int er_fm_block_bwd(const float* x, const float* gy, const float* g_pass, const float* coef_dev,
                    float coef_mul, int64_t batch, int32_t n_field, int32_t dim, int32_t x_stride,
                    int32_t g_pass_stride, float* gx, int32_t gx_stride, er_stream_t stream);

/* Column concat into a pitched matrix and its gradient (tf.concat(axis=1), model/deepfm.py:76):
 * dst[b, first_i + c] = srcs[i][b, c]; columns past the last piece up to dst_stride are written as 0.
 * er_split_cols scatters the columns of src back into the pieces. */
#define ER_MAX_CAT 8
int er_concat_cols(const float* const* srcs, const int32_t* widths, const int32_t* strides, int32_t n,
                   int64_t batch, float* dst, int32_t dst_stride, er_stream_t stream);
int er_split_cols(const float* src, int32_t src_stride, int64_t batch, float* const* dsts,
                  const int32_t* widths, const int32_t* strides, int32_t n, er_stream_t stream);

/* Wide block (model/deepfm.py:62-63 and the regulariser of layers/input_layer.py:369-375):
 *   fwd: y[b] = sum_f x[b,f]; *sumsq_out = sum x^2 (NULL: skipped; ws as er_fm_block_fwd)
 *   bwd: gx[b,f] = gy[b] + (*coef_dev * coef_mul) * x[b,f] */
int er_rowsum_block_fwd(const float* x, int64_t batch, int32_t width, int32_t x_stride, float* y,
                        float* sumsq_out, void* ws, size_t ws_bytes, er_stream_t stream);
int er_rowsum_block_bwd(const float* x, const float* gy, const float* coef_dev, float coef_mul,
                        int64_t batch, int32_t width, int32_t x_stride, float* gx, int32_t gx_stride,
                        er_stream_t stream);

/* Single-unit dense head (the logit layer tf.layers.dense(units=1), model/deepfm.py:75-105,
 * rank_model.py:57-74): y[b] = x[b,:].w + bias;  gx[b,f] = g[b]*w[f] (gx NULL: skipped),
 * gw[f] = sum_b g[b]*x[b,f], gb = sum_b g[b] (deterministic).  ws: er_dense1_workspace_bytes(width),
 * first 16 bytes zero on first use (left zero). */
size_t er_dense1_workspace_bytes(int32_t width);
int er_dense1_fwd(const float* x, const float* w, const float* bias, int64_t batch, int32_t width,
                  int32_t x_stride, float* y, er_stream_t stream);
int er_dense1_bwd(const float* x, const float* w, const float* g, int64_t batch, int32_t width,
                  int32_t x_stride, float* gx, int32_t gx_stride, float* gw, float* gb, void* ws,
                  size_t ws_bytes, er_stream_t stream);

/* ---- K6 epilogues: dense bias + batch-norm + relu (layers/dnn.py:56-79) ------
 * z is the SGEMM output x W (no bias).  Training: batch statistics (biased
 * variance, tf.layers.batch_normalization defaults) are computed deterministically
 * in two launches; moving_mean / moving_var are updated with `momentum`.
 * gamma == NULL means "no batch norm": y = act(z + bias).
 * ws: er_dense_workspace_bytes(batch, units). */
size_t er_dense_workspace_bytes(int64_t batch, int32_t units);
int er_bias_bn_act_fwd(const float* z, const float* bias, const float* gamma,
                       const float* beta, float* moving_mean, float* moving_var,
                       int64_t batch, int32_t units, float eps, float momentum,
                       int32_t training, int32_t relu, float* y, float* save_mean,
                       float* save_rstd, void* ws, size_t ws_bytes,
                       er_stream_t stream);
/* gz = dL/dz; ggamma/gbeta = batch-norm parameter gradients; gbias = column sum
 * of gz (identically zero under batch norm). */
int er_bias_bn_act_bwd(const float* z, const float* bias, const float* gamma,
                       const float* y, const float* gy, const float* save_mean,
                       const float* save_rstd, int64_t batch, int32_t units,
                       int32_t relu, float* gz, float* gbias, float* ggamma,
                       float* gbeta, void* ws, size_t ws_bytes, er_stream_t stream);
/* The same backward for batch norm + relu (gamma and beta given), with the relu mask recomputed from z - y > 0 exactly
 * when ((z + bias - mean) * rstd * gamma + beta) > 0 in the forward kernels' rounding - so y is not read.  Two launches
 * (column sums, then gz), ws: er_dense_workspace_bytes; units % 4 == 0 and every array 16-byte aligned. */
int er_bn_relu_bwd(const float* z, const float* bias, const float* gamma, const float* beta,
                   const float* save_mean, const float* save_rstd, const float* gy, int64_t batch, int32_t units,
                   int32_t relu, float* gz, float* gbias, float* ggamma, float* gbeta, void* ws, size_t ws_bytes,
                   er_stream_t stream);

/* tf.nn.dropout of DNN.__call__ (layers/dnn.py:77-82): y = x * mask / (1 - rate), mask ~ Bernoulli(1 - rate) per
 * element, a counter-based function of (seed, *counter_dev, element index): element i is kept iff the top 32 bits of
 * the splitmix64 finaliser of seed + counter * 0x9E3779B97F4A7C15 + i * 0xD1B54A32D192ED03 are below
 * floor((1 - rate) * 2^32), so rate 0 keeps every element; a kept value is x * fp32(1 / (1 - rate)).  The backward
 * pass is the SAME call on the upstream gradient (same seed, same counter value): the mask is recomputed, not stored.
 * counter_dev is a device
 * int64 the caller advances once per step, so a captured graph draws a new mask on every replay. */
int er_dropout(const float* x, int64_t n, float rate, uint64_t seed, const int64_t* counter_dev, float* y,
               er_stream_t stream);

/* The stateless non-relu activations of get_activation (utils/activation.py:66-118), applied by DNN.__call__
 * (layers/dnn.py:70-73) and the keras MLP block (layers/keras/blocks.py:82) after the dense / batch-norm stage:
 * y = f(x) elementwise; the backward pass recomputes f'(x) from the pre-activation: gx = gy * f'(x).  relu stays fused
 * in er_bias_bn_act_*; 'linear' is no call at all; dice (learned alpha over a batch norm): er_dice_* below. */
enum {
  ER_ACT_GELU = 1,       /* x * 0.5 * (1 + tanh(sqrt(2/pi) * (x + 0.044715 x^3)))  (activation.py:46-60) */
  ER_ACT_LEAKY_RELU = 2, /* tf.nn.leaky_relu, alpha 0.2 (also 'prelu' without arguments, activation.py:98-101) */
  ER_ACT_ELU = 3,
  ER_ACT_SELU = 4,
  ER_ACT_TANH = 5,
  ER_ACT_SWISH = 6,      /* x * sigmoid(x) */
  ER_ACT_SIGMOID = 7
};
int er_act_fwd(const float* x, int64_t n, int kind, float* y, er_stream_t stream);
int er_act_bwd(const float* x, const float* gy, int64_t n, int kind, float* gx, er_stream_t stream);

/* dice (utils/activation.py:13-43; layers/keras/activation.py:24-73), the data-adaptive activation of DIN:
 * y = alpha[c] * (1 - p) * x + p * x with p = sigmoid(xn), xn = batch_norm(x) WITHOUT centre / scale and epsilon 1e-9
 * (the caller runs it with er_bias_bn_act_fwd on unit gamma / zero beta; moving statistics, momentum 0.99).  x, xn, y:
 * [batch, units]; alpha [units].  Backward: gx_direct = gy * (alpha (1 - p) + p), gxn = gy * x * (1 - alpha) * p (1 - p)
 * (the caller continues it through er_bias_bn_act_bwd and adds the result to gx_direct), galpha_terms[b, c] = gy * x *
 * (1 - p) (summed over b by the caller). */
int er_dice_fwd(const float* x, const float* xn, const float* alpha, int64_t batch, int32_t units, float* y,
                er_stream_t stream);
int er_dice_bwd(const float* x, const float* xn, const float* alpha, const float* gy, int64_t batch, int32_t units,
                float* gx_direct, float* gxn, float* galpha_terms, er_stream_t stream);

/* One batch into the accumulators of tf.metrics.auc (model/rank_model.py:360-373; eval.proto AUC.num_thresholds,
 * default 200) and max_f1 (core/metrics.py:25-56).  thresholds: DEVICE float32[n_thresholds], ascending (TF's list:
 * -1e-7, (i + 1) / (T - 1) for i < T - 2, 1 + 1e-7).  hist: DEVICE uint64[2 * (n_thresholds + 1)], zeroed by the caller
 * before the first batch; hist[k] counts the negatives and hist[n_thresholds + 1 + k] the positives (int64(label) != 0)
 * whose prediction exceeds exactly k thresholds, so tp[i] = sum_{k > i} pos[k], fp[i] = sum_{k > i} neg[k].  Integer
 * counters: exact and independent of the order of the batches. */
int er_auc_hist(const float* probs, const float* labels, int64_t n, const float* thresholds, int32_t n_thresholds,
                uint64_t* hist, er_stream_t stream);

/* Dense optimizer over ONE flat parameter buffer (dense apply_gradients,
 * compat/optimizers.py:413-416): g = grad*grad_scale + l2*w, then the adagrad / adam / sgd rule.
 * segs: DEVICE array describing the tensors inside the flat buffers; the step's rate is lr_dev when given
 * (optional device scalar: the effective rate, used as is, also for Adam).  Otherwise lr and Adam's beta
 * powers come from opt->hyper_dev (device memory, so a captured CUDA graph can follow a schedule) or, when
 * that is NULL, from opt->lr, opt->beta1_power and opt->beta2_power; for the Adam kinds the kernel forms
 * lr_t = lr*sqrt(1-b2^t)/(1-b1^t) from them, as er_embedding_bwd and er_sparse_apply do.  grad_scale always
 * comes from opt->grad_scale, never from hyper_dev: the dense and the sparse gradients scale differently.
 * The rate of a segment is that rate times its lr_mult.  reg_loss_out (optional) += sum l2/2*w^2 of the
 * pre-update weights (float atomics: not bit-reproducible). */
typedef struct er_dense_seg {
  int64_t offset;
  int64_t n;
  float l2;
  float lr_mult;
} er_dense_seg_t;
int er_dense_apply(float* params, const float* grads, float* state0, float* state1,
                   const er_dense_seg_t* segs, int32_t n_segs, int64_t max_seg_n,
                   const er_opt_t* opt, const float* lr_dev, float* reg_loss_out,
                   er_stream_t stream);

/* ---- dense-layer GEMM on the Hopper tensor cores (wgmma) (layers/dnn.py:50-87 tf.layers.dense and its
 * gradient): C[M,N] = A(M,K).B(K,N) (+ bias[n]), fp32 in / fp32 accumulate / fp32 out, operands split
 * hi+lo into three TF32 products ("3xTF32", error ~1e-6 relative - inside the 1e-4 logit budget).
 * Operands are read where they lie:
 *   a_mn_major = 0: A is [M, lda] with k contiguous      a_mn_major = 1: A is [K, lda] with m contiguous
 *   b_mn_major = 0: B is [N, ldb] with k contiguous      b_mn_major = 1: B is [K, ldb] with n contiguous
 * so forward (X, W[in,out]) = (0,1), dX (dY, W) = (0,0), dW (X, dY) = (1,1) need no transposed copy.
 * Pitches must be multiples of 4 floats and at least the row (lda >= K resp. M, ldb >= K resp. N, ldc >= N),
 * and base pointers of A and B 16-byte aligned (K, M, N are free; C may be pitched and misaligned).
 * Small-output / long-K problems are split along K; partials go to ws (er_gemm_workspace_bytes) and
 * are summed in a fixed order (deterministic). */
size_t er_gemm_workspace_bytes(int64_t M, int64_t N, int64_t K);
int er_gemm(const float* A, int64_t lda, int32_t a_mn_major, const float* B, int64_t ldb,
            int32_t b_mn_major, const float* bias, float* C, int64_t ldc, int64_t M, int64_t N,
            int64_t K, void* ws, size_t ws_bytes, er_stream_t stream);

/* Vector-sized dense layers: C[M,N] = A(M,K).B(K,N) (+ bias[n]) when one of M, N, K is below 8 - the MMoE gate
 * layers dense(x) -> [B, num_expert] (layers/mmoe.py:66-72) with their dX and dW - where a 128 x 128 tensor-core tile
 * would be almost all padding.  CUDA cores, fp32 FMA in k order; A(m,k) = A[m*sa_m + k*sa_k], B(k,n) = B[k*sb_k +
 * n*sb_n] (any strides, in floats: transposed views are read in place).  A long K over few outputs (the dW form, K =
 * batch) is cut into slices whose partials go to ws (er_gemm_small_workspace_bytes, 0 when unsplit) and are summed in
 * slice order: deterministic. */
size_t er_gemm_small_workspace_bytes(int64_t M, int64_t N, int64_t K);
int er_gemm_small(const float* A, int64_t sa_m, int64_t sa_k, const float* B, int64_t sb_k, int64_t sb_n,
                  const float* bias, float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, void* ws, size_t ws_bytes,
                  er_stream_t stream);

/* Dense + batch-norm training forward: the GEMM also produces the batch statistics of its output
 * columns (per-tile Welford partials merged in tile order by the last CTA of each column tile:
 * deterministic, no extra pass over z).  On return (stream order) save_mean[n] = mean(z[:,n]) + bias[n],
 * save_rstd[n] = 1/sqrt(biased var + eps) and, when given, the moving statistics are updated with
 * `momentum` (tf.layers.batch_normalization, layers/dnn.py:64-72).  z itself is stored WITHOUT the bias;
 * er_bn_act_apply adds it.  Needs an unsplit K (er_gemm_workspace_bytes(M,N,K) == 0) and a workspace of
 * er_gemm_bn_workspace_bytes(M,N) whose first 1024 bytes are zero on first use (left zero afterwards). */
typedef struct {
  const float* bias;      /* [N] or NULL */
  float* save_mean;       /* [N] out */
  float* save_rstd;       /* [N] out */
  float* moving_mean;     /* [N] in/out or NULL */
  float* moving_var;      /* [N] in/out or NULL */
  float eps;
  float momentum;
} er_bn_stats_t;
size_t er_gemm_bn_workspace_bytes(int64_t M, int64_t N);
int er_gemm_bn(const float* A, int64_t lda, int32_t a_mn_major, const float* B, int64_t ldb,
               int32_t b_mn_major, float* C, int64_t ldc, int64_t M, int64_t N, int64_t K,
               const er_bn_stats_t* bn, void* ws, size_t ws_bytes, er_stream_t stream);
/* Pre-split B operands (the dense towers' weights, split once per step instead of once per 128-row output tile).
 * er_gemm_split_planes writes, for each job, src(row, k) = src[row*ld_row + k*ld_k] (rows x k, any strides) as
 * hi = tf32(x) and lo = x - hi planes of er_gemm_plane_floats(rows, k) floats each, in the K-major swizzled tile order
 * er_gemm_planes reads, zero-padded to whole tiles; hi / lo 16-byte aligned.  One launch per 32 jobs.
 * er_gemm_planes is er_gemm (bn NULL) or er_gemm_bn (bn given, bias NULL) with B given as the planes of its
 * [N x K] K-major form (rows = N): forward of a dense layer W[in,out] -> the planes of W^T (ld_row 1, ld_k out),
 * dX -> the planes of W (ld_row out, ld_k 1).  The products are bit-identical to er_gemm / er_gemm_bn on B. */
typedef struct {
  const float* src;
  int64_t ld_row, ld_k;   /* in floats */
  int64_t rows, k;
  float* hi;
  float* lo;
} er_gemm_plane_t;
size_t er_gemm_plane_floats(int64_t rows, int64_t K);
int er_gemm_split_planes(const er_gemm_plane_t* planes, int32_t n, er_stream_t stream);
int er_gemm_planes(const float* A, int64_t lda, int32_t a_mn_major, const float* b_hi, const float* b_lo,
                   const float* bias, float* C, int64_t ldc, int64_t M, int64_t N, int64_t K,
                   const er_bn_stats_t* bn, void* ws, size_t ws_bytes, er_stream_t stream);
/* y = act((z + bias - mean) * rstd * gamma + beta) with given statistics (one elementwise pass). */
int er_bn_act_apply(const float* z, const float* bias, const float* gamma, const float* beta,
                    const float* mean, const float* rstd, int64_t batch, int32_t units, int32_t relu,
                    float* y, er_stream_t stream);

/* sigmoid cross entropy (tf.losses.sigmoid_cross_entropy,
 * builders/loss_builder.py:36-39): *loss_out = inv_count * sum_b w*(max(x,0)-x*z+log1p(exp(-|x|)))
 * (assigned, not added to), probs[b] = sigmoid(x), g_logits[b] = w*(sigmoid(x)-z)*inv_count.
 * weights NULL: w = 1; loss_out / probs / g_logits NULL: not written.  One CTA, deterministic. */
int er_sigmoid_ce_fwd_bwd(const float* logits, const float* labels,
                          const float* weights, int64_t batch, float inv_count,
                          float* loss_out, float* probs, float* g_logits,
                          er_stream_t stream);

/* ---- K4: DIN target attention (layers/sequence_feature_layer.py:150-189,
 * model/multi_tower_din.py:62-97).  The attention MLP is a library SGEMM chain; these are the
 * fused pieces around it:
 *  concat: din_in[b,t,:] = [q, k, q-k, q*k]  ([B*T, 4D]) and its backward
 *  pool  : scores[B,T] masked at t >= len with -2^32+1, softmax over T,
 *          out[b,:] = sum_t p[b,t]*keys[b,t,:]; backward routes no gradient to padded scores */
int er_din_concat_fwd(const float* query, const float* keys, int64_t batch,
                      int32_t seq_len, int32_t dim, float* din_in, er_stream_t stream);
int er_din_concat_bwd(const float* query, const float* keys, const float* g_din_in,
                      int64_t batch, int32_t seq_len, int32_t dim, float* g_query,
                      float* g_keys, int32_t accumulate_gkeys, er_stream_t stream);
int er_din_pool_fwd(const float* scores, const float* keys, const int32_t* lens,
                    int64_t batch, int32_t seq_len, int32_t dim, float* probs,
                    float* out, er_stream_t stream);
int er_din_pool_bwd(const float* probs, const float* keys, const float* gout,
                    const int32_t* lens, int64_t batch, int32_t seq_len, int32_t dim,
                    float* g_scores, float* g_keys, int32_t accumulate_gkeys,
                    er_stream_t stream);
/* sigmoid pool (attention_normalizer 'sigmoid' of the keras DIN block, layers/keras/din.py:57-60), the
 * arguments of er_din_pool_* plus `scale` (1/sqrt(history width) there):
 *   probs[b,t] = t < len ? sigmoid(scale*scores[b,t]) : 0, out[b,:] = sum_t probs[b,t]*keys[b,t,:]
 *   (ascending t, deterministic);
 *   bwd: g_scores[b,t] = t < len ? scale*p*(1-p)*(gout[b,:].keys[b,t,:]) : 0,
 *        g_keys[b,t,:] (+)= p*gout[b,:].  lens NULL: every step counts. */
int er_din_sigmoid_pool_fwd(const float* scores, const float* keys, const int32_t* lens,
                            int64_t batch, int32_t seq_len, int32_t dim, float scale,
                            float* probs, float* out, er_stream_t stream);
int er_din_sigmoid_pool_bwd(const float* probs, const float* keys, const float* gout,
                            const int32_t* lens, int64_t batch, int32_t seq_len, int32_t dim,
                            float scale, float* g_scores, float* g_keys,
                            int32_t accumulate_gkeys, er_stream_t stream);

/* ---- K5: DCN cross layer (model/dcn.py:32-45): out = x0*(xl.w) + b + xl; xw_out[b] = xl.w.
 * bwd: gxl = gout + w*s, gx0 (+)= gout*xw, gw = sum_b s_b*xl[b,:], gb = sum_b gout[b,:]
 * with s_b = gout[b,:].x0[b,:] (deterministic two-stage column sums).
 * ws: er_cross_workspace_bytes(batch, dim). */
int er_cross_fwd(const float* x0, const float* xl, const float* w, const float* b,
                 int64_t batch, int32_t dim, float* out, float* xw_out,
                 er_stream_t stream);
size_t er_cross_workspace_bytes(int64_t batch, int32_t dim);
int er_cross_bwd(const float* x0, const float* xl, const float* w, const float* xw,
                 const float* gout, int64_t batch, int32_t dim, float* gx0, float* gxl,
                 float* gw, float* gb, int32_t accumulate_gx0, void* ws, size_t ws_bytes,
                 er_stream_t stream);

/* ---- MMoE mixture (layers/mmoe.py:73-83): out[b,:] = sum_e softmax(gate[b,:])[e]*experts[b,e,:] */
int er_mmoe_mix_fwd(const float* gate_logits, const float* experts, int64_t batch,
                    int32_t n_expert, int32_t dim, float* probs, float* out,
                    er_stream_t stream);
int er_mmoe_mix_bwd(const float* probs, const float* experts, const float* gout,
                    int64_t batch, int32_t n_expert, int32_t dim, float* g_gate_logits,
                    float* g_experts, int32_t accumulate_gexperts, er_stream_t stream);

/* ---- DSSM (model/dssm.py:64-71, model/match_model.py:50-69,213-234) ----
 * l2norm: tf.nn.l2_normalize rows, y = x * rsqrt(max(sum x^2, 1e-12)), inv_norm[b] = that rsqrt.  A row with
 * sum x^2 < 1e-12f gets inv_norm = 1e6f exactly (1/sqrt(1e-12f) in fp32) and the clamped gradient gx = gy*inv_norm;
 * other rows get gx = inv_norm*(gy - y*(gy.y)).  The backward picks the branch by inv_norm == 1e6f, so rows with
 * sum x^2 at 1e-12f or a few ulp above it (where rsqrtf also gives 1e6f) take the clamped gradient too.
 * inbatch_softmax_ce: rows of sim [B, n_cols >= B], the
 * positive of row b is column b, in-batch duplicates of its item id are masked with -1e32,
 * loss_rows[b] = -log(p_bb + 1e-12)*w_b*inv_wsum (sum them for the loss), g_sim = dloss/dsim. */
int er_l2norm_fwd(const float* x, int64_t batch, int32_t dim, float* y, float* inv_norm,
                  er_stream_t stream);
int er_l2norm_bwd(const float* y, const float* inv_norm, const float* gy, int64_t batch,
                  int32_t dim, float* gx, er_stream_t stream);
int er_inbatch_softmax_ce(const float* sim, const int64_t* item_ids, const float* weights,
                          int64_t batch, int32_t n_cols, float inv_wsum, float* loss_rows,
                          float* probs_diag, float* g_sim, er_stream_t stream);

/* ---- DLRM / DotInteraction pairwise dot products (model/dlrm.py:52-61 `einsum('bne,bme->bnm')`,
 * layers/keras/interaction.py:47-128): out[b,i,j] = x[b,i,:].x[b,j,:] for x [B, n, dim] (contiguous);
 * gx[b,i,:] = sum_j (g[b,i,j] + g[b,j,i]) * x[b,j,:].  Sequential sums: deterministic. */
int er_gram_fwd(const float* x, int64_t batch, int32_t n, int32_t dim, float* out, er_stream_t stream);
int er_gram_bwd(const float* x, const float* g, int64_t batch, int32_t n, int32_t dim, float* gx,
                er_stream_t stream);

/* ---- CSV input: text lines -> the column arrays of the packed batch (HOST function, HOST pointers) ----
 * Replaces tf.decode_csv + the per-field parsing of the CSV input path (input/csv_input.py:78-175,
 * input/input.py:537-675: ids stay int64 / string ids are fingerprinted, raw values become fp32, Tag /
 * Sequence fields are split on their inner separator).  Empty or missing fields take the column default
 * (record_defaults).  No quoting.  Parses the complete lines of buf[0, len) up to max_rows; *consumed is
 * the offset of the first unparsed byte (an unterminated last line stays with the caller). */
enum {
  ER_CSV_SKIP = 0,
  ER_CSV_I64 = 1,      /* out int64[max_rows]: decimal integer */
  ER_CSV_F32 = 2,      /* out float[max_rows] */
  ER_CSV_HASH = 3,     /* out int64[max_rows]: Fingerprint64 of the field bytes (string-typed id field);
                          with hash_mod: Fingerprint64 % hash_mod as uint64 (string_to_hash_bucket_fast,
                          feature_column_v2.py:3915-3921) and -1 for an empty string (dropped by the lookup) */
  ER_CSV_I64_LIST = 4, /* out int64[list_cap] + lens int32[max_rows]: inner_sep-separated integers, empty
                          tokens dropped, at most `width` per line when width > 0 (the first ones) */
  ER_CSV_F32_VEC = 5,  /* out float[max_rows * width]: inner_sep-separated floats, zero padded */
  ER_CSV_HASH_LIST = 6, /* like ER_CSV_I64_LIST, every token fingerprinted (string Tag / Sequence tokens) */
  ER_CSV_I64_KV_LIST = 7,  /* tokens `key<kv_sep>weight` (TagFeature kv_separator, input/input.py:447-458): integer
                              keys to out, fp32 weights to `weights` at the same positions */
  ER_CSV_HASH_KV_LIST = 8, /* the same with fingerprinted string keys */
  ER_CSV_F32_LIST = 9,     /* out float[list_cap] + lens int32[max_rows]: inner_sep-separated floats, empty tokens
                            * skipped - the weight input of a TagFeature (its second input_names entry,
                            * input/input.py:477-497) */
  ER_CSV_I64_STEP_LIST = 10, /* SequenceFeature with seq_multi_sep (input/input.py:686-700): steps separated by
                            * inner_sep, the values of one step by kv_sep.  out int64[list_cap] = the values of all
                            * steps back to back, lens[r] = steps of line r (the first `width` non-empty ones),
                            * step_lens int32[max_rows * width] = values per step (0 beyond lens[r]) */
  ER_CSV_HASH_STEP_LIST = 11, /* the same with fingerprinted string values */
  ER_CSV_F64 = 12          /* out double[max_rows]: a decimal number (strtod on the field without its surrounding
                            * spaces / tabs; hex spellings are refused), an ExprFeature input read from a STRING or
                            * DOUBLE field (tf.string_to_number(.., tf.float64), input/input.py:513-523).  An empty
                            * field parses default_str instead; NULL or "" there makes an empty field invalid */
};
typedef struct {
  int32_t kind;
  int32_t width;
  char inner_sep;
  char kv_sep;             /* key / weight separator of the *_KV_LIST kinds */
  char pad_[6];
  int64_t default_i64;
  float default_f32;
  int32_t pad2_;
  const char* default_str; /* ER_CSV_HASH: hashed instead of an empty field (NULL = "") */
  void* out;
  int32_t* lens;
  int64_t list_cap;
  int64_t n_vals;          /* written by the call: values stored for a list column */
  uint64_t hash_mod;       /* ER_CSV_HASH / ER_CSV_HASH_LIST: 0 = raw fingerprints, else the hash_bucket_size */
  float* weights;          /* *_KV_LIST: float[list_cap] */
  int32_t* step_lens;      /* *_STEP_LIST: int32[max_rows * width] */
} er_csv_col_t;
int er_csv_parse(const char* buf, size_t len, char sep, er_csv_col_t* cols, int32_t n_cols,
                 int64_t max_rows, int32_t n_threads, int64_t* n_rows, size_t* consumed);
/* The same parse over every line_stride-th line of the buffer, from line line_phase on (0 <= line_phase <
 * line_stride): the rows are the kept lines only, in buffer order; every newline is scanned but only kept lines are
 * split into fields.  *lines_seen = complete lines passed over up to *consumed (kept or not).  Rank r of N reading
 * lines r::N of a file passes line_stride = N and the phase of its next line.  er_csv_parse is line_stride 1. */
int er_csv_parse_lines(const char* buf, size_t len, char sep, er_csv_col_t* cols, int32_t n_cols,
                       int64_t max_rows, int32_t n_threads, int64_t line_stride, int64_t line_phase,
                       int64_t* n_rows, size_t* consumed, int64_t* lines_seen);

/* Fingerprint64 of the decimal text of each int64 (tf.as_string + the string hash): what an integer input of a
 * crossed / hashed column contributes (input/input.py:356-376).  HOST pointers. */
int er_fingerprint64_i64(const int64_t* values, int64_t n, uint64_t* out);

/* ---- CriteoInput batches (input/criteo_binary_reader.py, input/criteo_input.py:76-86) ----
 * One batch of the binary parts, as read from the files: label int32[batch], dense float32[batch, 13] and cat
 * uint32[batch, 26], row-major.  Writes the batch form of the other readers:
 *   sparse_fea int64[n_slot * batch], feature-major: sparse_fea[s * batch + b] = (int64)(int32) cat[b, slot_cols[s]]
 *     (the reference's declared tf.int32 output type);
 *   dense_fea float32[batch, n_raw]: dense_fea[b, j] = dense[b, raw_cols[j]];
 *   labels float32[batch] = (float) label.
 * slot_cols int32[n_slot] (duplicates allowed) and raw_cols int32[n_raw] are DEVICE arrays whose entries the caller
 * keeps in [0, 26) and [0, 13): they live in device memory, where this call cannot check them.  n_slot 0 / n_raw 0 skip
 * that output (its pointers may then be null).  No allocation, no synchronisation. */
#define ER_CRITEO_N_DENSE 13
#define ER_CRITEO_N_CAT 26
int er_binary_unpack(const int32_t* label, const float* dense, const uint32_t* cat, int64_t batch,
                     const int32_t* slot_cols, int32_t n_slot, const int32_t* raw_cols, int32_t n_raw,
                     int64_t* sparse_fea, float* dense_fea, float* labels, er_stream_t stream);

/* ---- ExprFeature columns (input/input.py:507-535, utils/expr_util.py) ----
 * Each expression of a model is a postfix program over the float64 inputs of one sample, compiled on the host
 * (easyrec_b200/expr.py).  An op pushes an input (ER_EXPR_LOAD, arg = input index) or a constant (ER_EXPR_CONST, value),
 * negates the top (ER_EXPR_NEG), or pops two values a (below) and b (top) and pushes a op b: + - * / in float64
 * rounded to nearest, the five comparisons and & / | (operands 0.0 = false, else true) as 1.0 / 0.0. */
#define ER_EXPR_MAX_STACK 8      /* values on the evaluation stack */
#define ER_EXPR_MAX_OPS 4096     /* ops of all the programs of one call */
enum {
  ER_EXPR_LOAD = 0, ER_EXPR_CONST = 1, ER_EXPR_ADD = 2, ER_EXPR_SUB = 3, ER_EXPR_MUL = 4, ER_EXPR_DIV = 5,
  ER_EXPR_NEG = 6, ER_EXPR_GT = 7, ER_EXPR_GE = 8, ER_EXPR_LT = 9, ER_EXPR_LE = 10, ER_EXPR_EQ = 11,
  ER_EXPR_AND = 12, ER_EXPR_OR = 13
};
typedef struct {
  int32_t op;
  int32_t arg;
  double value;
} er_expr_op_t;          /* 16 bytes */
typedef struct {
  int32_t begin;         /* first op of the program in the ops array */
  int32_t n_ops;
  int32_t out_col;       /* the column of dense the result goes to */
  int32_t pad_;
} er_expr_t;             /* 16 bytes */
/* dense[b * dense_pitch + exprs[e].out_col] = (float) (value of program e on inputs[b * n_inputs ...]) for every sample
 * b < batch and expression e < n_expr: one launch, one thread per (expression, sample).  inputs float64[batch,
 * n_inputs], exprs er_expr_t[n_expr] and ops er_expr_op_t[n_ops] are DEVICE arrays (exprs and ops may be one
 * allocation).  max_depth: the deepest stack any program needs, at most ER_EXPR_MAX_STACK; a program that goes deeper
 * loses its bottom values.  The kernel reads only inside the arrays it is given whatever they hold: an input index
 * outside [0, n_inputs) reads NaN, a program reaching past n_ops runs no op, an out_col outside [0, dense_pitch) writes
 * nothing.  No allocation, no synchronisation; capturable in a CUDA graph. */
int er_expr_eval(const double* inputs, int64_t batch, int32_t n_inputs, const er_expr_t* exprs, int32_t n_expr,
                 const er_expr_op_t* ops, int32_t n_ops, int32_t max_depth, float* dense, int64_t dense_pitch,
                 er_stream_t stream);

/* ---- sharded-table restore: the LoadEmbed custom op (ops/src/load_dense_embed.cc:28-156;
 * python fallback compat/embedding_parallel_saver.py:141-173) ----
 * HOST function, HOST pointers (the op is a CPU kernel in the reference as well).  Reads every
 * `<ckpt_path>-embedding/<var_name>-part-<p>.bin` (raw fp32 [rows_p, embed_dim]; row j of old part p
 * is global row j * P + p, P = number of part files), and fills this worker's shard
 * vals[embed_part_size, embed_dim]: global rows g with g % task_num == task_index and
 * g < embed_part_size * task_num land on local row g / task_num; rows no file provides stay 0.
 * var_name is the file stem the saver used ("embed-" + variable name with '/' -> "__").
 * *rows_loaded (optional) receives the number of rows copied; like the op, anything but
 * embed_part_size or embed_part_size - 1 is an error (ER_ERR_INVALID_ARG). */
int er_load_embed(const char* ckpt_path, const char* var_name, int32_t task_index, int32_t task_num,
                  int32_t embed_dim, int64_t embed_part_size, float* vals, int64_t* rows_loaded);

/* ---- key-value embedding tables (ev_params; feature_column/feature_column.py:250-256,288-291, SOK DynamicVariable at
 * compat/feature_column/feature_column.py:425-503) ----
 * A KV table's slots have num_buckets = 2^63 - 1, so K1 writes the KEY (>= 0, or -1 for a dropped lookup) where a
 * static table has its row.  These calls turn keys into rows of a pool of `capacity` rows through an open-addressing
 * index: index_keys int64[n_index] (every entry ER_KV_EMPTY before first use) and index_rows int64[n_index], n_index a
 * power of two >= 16 and >= 2 * capacity.  stats int64[2]: [0] rows handed out so far (may pass capacity: the keys
 * beyond it have no row), [1] live lookups that were left without a row.  The host reads stats outside the step.
 * Row numbers depend on the order of claims and are not deterministic; nothing else does.  No allocation, no host
 * synchronisation, and no thread waits on another thread's store. */
#define ER_KV_EMPTY (-1)

/* Training lookup: find-or-insert.  The key of lookup l is keys[l] * shard_n + shard_rank (keys[l] < 0: none): a
 * row-sharded table's owner passes the owner-local keys it received (K1's key div N) and its rank, an unsharded table
 * 1 and 0.  rows[l] = the pool row of that key (-1 without a key or when the pool has no row left for it).  A key seen
 * for the first time is claimed in the index and, while the pool has rows, gets the next one, initialised: weight[row,
 * c] = a normal(0, init_stddev), truncated at 2 init_stddev when init_truncated, drawn from a counter-based hash of
 * (seed, key, c); state0 (may be null) = state0_init and state1 (may be null) = 0 over the row's dim columns.  weight /
 * state0 / state1 share row_stride (floats).  Two launches: claim and initialise, then resolve.  keys and rows must
 * not alias. */
int er_kv_find_or_insert(int64_t* index_keys, int64_t* index_rows, int64_t n_index, int64_t capacity,
                         int64_t* stats, const int64_t* keys, int64_t n, int32_t shard_n, int32_t shard_rank,
                         int64_t* rows, float* weight, float* state0, float* state1, int64_t row_stride, int32_t dim,
                         float state0_init, uint64_t seed, float init_stddev, int32_t init_truncated,
                         er_stream_t stream);
/* Evaluation / prediction lookup: find only, keys as in er_kv_find_or_insert.  rows[l] = the row of the key; a key
 * without a row reads zero_row (a row the caller keeps at zero: "new key will get zero embedding",
 * feature_column_v2.py:3489-3494); keys[l] < 0 -> -1. */
int er_kv_find(const int64_t* index_keys, const int64_t* index_rows, int64_t n_index, const int64_t* keys,
               int64_t n, int32_t shard_n, int32_t shard_rank, int64_t zero_row, int64_t* rows, er_stream_t stream);
/* Restore: insert keys[i] with the given row rows[i], for distinct keys >= 0 into an empty index (2 * n <= n_index).  A
 * negative or repeated key counts in stats[1]; stats[0] is the caller's to set. */
int er_kv_insert_rows(int64_t* index_keys, int64_t* index_rows, int64_t n_index, const int64_t* keys,
                      const int64_t* rows, int64_t n, int64_t* stats, er_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* ER_B200_H_ */
