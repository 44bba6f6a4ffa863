// K0: lens -> CSR (row_ptr, seg_ids);  K1: raw int64 ids -> arena rows.
//
// Reference ops replaced (SURVEY.md section 2.5 K1):
//   cumsum(lens) + searchsorted        compat/feature_column/feature_column.py:264-266
//   as_string + string_to_hash_bucket_fast   feature_column_v2.py:3915-3921
//   vals % num_buckets                 input/parquet_input.py:221
//   identity column with default 0     feature_column_v2.py:4268-4292
//   uniq % N / int64(recv / N)         compat/feature_column/feature_column.py:296,317
//   vocabulary list / file, default 0  feature_column/feature_column.py:277-290,320-333,497-509
// The hashing kernels are pure streaming integer work: 8 B in + 8 B out per lookup; a vocabulary lookup adds the
// probe of its index (one or two 128-byte groups at the index's load factor of at most 1/2).
#include "common.cuh"
#include "hash.cuh"
#include "kv_index.cuh"
#include "scan.cuh"
#include "slots.cuh"

namespace er {

struct LensIn {
  const int32_t* lens;
  __device__ int operator()(int64_t j) const { return lens[j]; }
};
struct RowPtrOut {
  int32_t* row_ptr;
  int64_t n;
  __device__ void operator()(int64_t j, int ex, int v) const {
    row_ptr[j] = ex;
    if (j == n - 1) row_ptr[n] = ex + v;
  }
};

__global__ void __launch_bounds__(256)
    expand_seg_ids_kernel(const int32_t* __restrict__ row_ptr, int64_t n_seg, int64_t cap,
                          int32_t* __restrict__ seg_ids) {
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < n_seg;
       s += (int64_t)gridDim.x * blockDim.x) {
    int64_t b = row_ptr[s], e = row_ptr[s + 1];
    if (e > cap) e = cap;
    for (int64_t j = b; j < e; ++j) seg_ids[j] = (int32_t)s;
  }
}

struct BucketRule {  // 32 bytes, staged in shared memory per CTA
  int64_t num_buckets;
  int64_t row_offset;
  int32_t seg_begin;
  int32_t mode;
  int32_t shard_n;
  int32_t combiner;  // er_combiner without the ER_COMBINER_UNIT_WEIGHTS flag
};

// Every CTA stages the slot plan's bucket rules in shared memory; returns whether the slots are uniform (slot f owns
// segments [f * n_seg, (f + 1) * n_seg)), in which case slot_rule() finds a segment's slot by a multiply-shift.
__device__ __forceinline__ int stage_rules(BucketRule* tab, const er_slot_t* __restrict__ slots, int n_slots) {
  const int nseg0 = slots[0].n_seg;
  int ok = 1;
  for (int i = threadIdx.x; i < n_slots; i += blockDim.x) {
    const er_slot_t s = slots[i];
    BucketRule r;
    r.num_buckets = s.num_buckets;
    r.row_offset = s.row_offset;
    r.seg_begin = s.seg_begin;
    r.mode = s.bucket_mode;
    r.shard_n = s.shard_n;
    r.combiner = s.combiner & 0xf;
    tab[i] = r;
    if (s.n_seg != nseg0 || s.seg_begin != i * nseg0) ok = 0;
  }
  return __syncthreads_and(ok);
}

__device__ __forceinline__ int slot_rule(const BucketRule* tab, int n_slots, int uniform, const FastDiv& div, int32_t s) {
  if (uniform) return (int)fastdiv((uint32_t)s, div);
  int lo = 0, hi = n_slots;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (tab[mid].seg_begin <= s)
      lo = mid;
    else
      hi = mid;
  }
  return lo;
}

// The bucket of one id under its slot's rule, before sharding and the table offset; `drop` is set for a lookup that
// reads no row.
__device__ __forceinline__ int64_t bucket_of(const BucketRule& t, int64_t v, bool& drop) {
  const int64_t nb = t.num_buckets;
  const int mode = t.mode;
  int64_t r;
  if (mode == ER_BUCKET_FARM_DECIMAL) {
    farm::Dec d = farm::to_decimal(v);
    uint64_t h = farm::fingerprint64_dec(d);
    r = (int64_t)(h % (uint64_t)nb);
  } else if (mode == ER_BUCKET_MOD) {
    int64_t m = v % nb;
    r = m < 0 ? m + nb : m;
  } else if (mode == ER_BUCKET_IDENTITY) {
    drop = (v == -1);
    r = (v < 0 || v >= nb) ? 0 : v;
  } else if (mode == ER_BUCKET_ONE_ROW) {
    drop = (v < 0);
    r = 0;
  } else {
    drop = (v < 0);
    r = v;
  }
  return r;
}

// rows[l] = table offset + (owner-local) row, owner[l] = bucket mod shard_n; -1 / -1 for a dropped lookup
__device__ __forceinline__ void store_row(const BucketRule& t, int64_t r, bool drop, int64_t l, int64_t* __restrict__ rows,
                                          int32_t* __restrict__ owner) {
  int32_t own = 0;
  if (t.shard_n > 1) {
    own = (int32_t)(r % t.shard_n);
    r = r / t.shard_n;
  }
  rows[l] = drop ? -1 : (t.row_offset + r);
  if (owner) owner[l] = drop ? -1 : own;
}

__global__ void __launch_bounds__(256)
    bucketize_kernel(const int64_t* __restrict__ ids, const float* __restrict__ weights,
                     const int32_t* __restrict__ seg_ids,
                     const int32_t* __restrict__ row_ptr, int64_t n_seg, int64_t cap,
                     const er_slot_t* __restrict__ slots, int n_slots,
                     int64_t* __restrict__ rows, int32_t* __restrict__ owner) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  BucketRule* tab = reinterpret_cast<BucketRule*>(s_raw);
  const int uniform = stage_rules(tab, slots, n_slots);
  const int nseg0 = slots[0].n_seg;
  const FastDiv div = make_fastdiv((uint32_t)(nseg0 > 0 ? nseg0 : 1));
  int64_t n = cap;
  if (row_ptr) {
    int64_t t = row_ptr[n_seg];
    n = t < cap ? t : cap;
  }
  for (int64_t l = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; l < n;
       l += (int64_t)gridDim.x * blockDim.x) {
    const int32_t s = seg_ids ? seg_ids[l] : (int32_t)l;
    const BucketRule& t = tab[slot_rule(tab, n_slots, uniform, div, s)];
    bool drop = false;
    const int64_t r = bucket_of(t, ids[l], drop);
    // _prune_invalid_weights (compat/embedding_ops.py): a mean / sqrtn lookup whose weight is not > 0 (NaN included)
    // is dropped here, so that K2, K7, er_mark_rows and K8 all see it as a dropped lookup
    if (weights && t.combiner != ER_COMBINER_SUM && !(weights[l] > 0.f)) drop = true;
    store_row(t, r, drop, l, rows, owner);
  }
}

// K1 over un-pooled histories: step l = (f * B + b) * T + t is segment l, and a step at or beyond its sample's length
// (lens[f * B + b]) reads no row.  Its id is not read at all, so the exchange of a row-sharded table never requests
// the padding.
__global__ void __launch_bounds__(256)
    bucketize_seq_kernel(const int64_t* __restrict__ ids, const int32_t* __restrict__ lens, int64_t n_steps, int T,
                         const er_slot_t* __restrict__ slots, int n_slots, int64_t* __restrict__ rows,
                         int32_t* __restrict__ owner) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  BucketRule* tab = reinterpret_cast<BucketRule*>(s_raw);
  er_pdl_wait();
  const int uniform = stage_rules(tab, slots, n_slots);
  const int nseg0 = slots[0].n_seg;
  const FastDiv div = make_fastdiv((uint32_t)(nseg0 > 0 ? nseg0 : 1));
  const FastDiv tdiv = make_fastdiv((uint32_t)T);
  for (int64_t l = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; l < n_steps;
       l += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t sample = fastdiv((uint32_t)l, tdiv);
    const int t_pos = (int)((uint32_t)l - sample * (uint32_t)T);
    if (t_pos >= lens[sample]) {   // (a length below 0 pads every step, one above T pads none)
      rows[l] = -1;
      if (owner) owner[l] = -1;
      continue;
    }
    const BucketRule& t = tab[slot_rule(tab, n_slots, uniform, div, (int32_t)l)];
    bool drop = false;
    const int64_t r = bucket_of(t, ids[l], drop);
    store_row(t, r, drop, l, rows, owner);
  }
}

// K1 for slot plans with vocabulary slots (ER_BUCKET_VOCAB); kSeq: the un-pooled history form of bucketize_seq_kernel.
// Each warp walks 32 consecutive lookups together (the loop bound is uniform over the warp, lanes past the end carry
// nothing), so its two 16-lane tiles are whole when they probe: a tile looks up its lanes' vocabulary keys one after
// the other, all 16 lanes comparing one 128-byte group of the index per step (kv_find_slot, csrc/kv_index.cuh).
// Lookups of the other modes take bucket_of as in the kernels above.
template <bool kSeq>
__global__ void __launch_bounds__(256)
    bucketize_vocab_kernel(const int64_t* __restrict__ ids, const float* __restrict__ weights,
                           const int32_t* __restrict__ seg_ids, const int32_t* __restrict__ row_ptr,
                           const int32_t* __restrict__ lens, int64_t n_seg, int64_t cap, int T,
                           const er_slot_t* __restrict__ slots, int n_slots, const er_vocab_t* __restrict__ vocabs,
                           int64_t* __restrict__ rows, int32_t* __restrict__ owner) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  BucketRule* tab = reinterpret_cast<BucketRule*>(s_raw);
  if constexpr (kSeq) er_pdl_wait();
  const int uniform = stage_rules(tab, slots, n_slots);
  const int nseg0 = slots[0].n_seg;
  const FastDiv div = make_fastdiv((uint32_t)(nseg0 > 0 ? nseg0 : 1));
  const FastDiv tdiv = make_fastdiv((uint32_t)T);
  int64_t n = cap;
  if (!kSeq && row_ptr) {
    const int64_t total = row_ptr[n_seg];
    n = total < cap ? total : cap;
  }
  const int lane = threadIdx.x & 31, t = lane & (kKvTile - 1), base = lane & kKvTile;
  const unsigned tmask = 0xFFFFu << base;
  for (int64_t l0 = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31); l0 < n;
       l0 += (int64_t)gridDim.x * blockDim.x) {
    const int64_t l = l0 + lane;
    bool live = l < n;
    int32_t s = (int32_t)l;
    if (live) {
      if constexpr (kSeq) {
        const uint32_t sample = fastdiv((uint32_t)l, tdiv);
        if ((int)((uint32_t)l - sample * (uint32_t)T) >= lens[sample]) {   // a padded step: its id is not read
          rows[l] = -1;
          if (owner) owner[l] = -1;
          live = false;
        }
      } else if (seg_ids) {
        s = seg_ids[l];
      }
    }
    const int f = live ? slot_rule(tab, n_slots, uniform, div, s) : 0;
    const int64_t v = live ? ids[l] : -1;
    const bool vocab = live && tab[f].mode == ER_BUCKET_VOCAB;
    bool drop = vocab && v < 0;
    int64_t r = 0;
    if (live && !vocab) r = bucket_of(tab[f], v, drop);
    // the tile's vocabulary keys, one at a time: a hit reads the entry's position, a miss row 0 (default_value 0)
    unsigned todo = (__ballot_sync(tmask, vocab && v >= 0) >> base) & 0xFFFFu;
    while (todo) {
      const int j = __ffs(todo) - 1;
      todo &= todo - 1;
      const int64_t k = __shfl_sync(tmask, v, base + j);
      const er_vocab_t vb = vocabs[__shfl_sync(tmask, f, base + j)];
      const KvIndex ix{(long long*)vb.index_keys, (int64_t*)vb.index_rows, vb.n_index / kKvTile};
      const int64_t e = kv_find_slot(ix, k, t, base, tmask);
      if (t == j) r = e >= 0 ? vb.index_rows[e] : 0;
    }
    if (!live) continue;
    const BucketRule& rule = tab[f];
    if (!kSeq && weights && rule.combiner != ER_COMBINER_SUM && !(weights[l] > 0.f)) drop = true;
    store_row(rule, r, drop, l, rows, owner);
  }
}

}  // namespace er

extern "C" size_t er_csr_workspace_bytes(int64_t n_seg) {
  return er::scan::workspace_bytes(n_seg);
}

extern "C" int er_csr_from_lens(const int32_t* lens, int64_t n_seg, int32_t* row_ptr,
                                int32_t* seg_ids, int64_t n_lookups_cap, void* ws,
                                size_t ws_bytes, er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(lens && row_ptr, "lens and row_ptr must be non-null");
  ER_REQUIRE(n_seg > 0 && n_seg < (1LL << 31), "n_seg out of range");
  ER_REQUIRE(n_lookups_cap >= 0 && n_lookups_cap < (1LL << 31), "n_lookups_cap out of range");
  if (ws_bytes < scan::workspace_bytes(n_seg) || !ws)
    return fail(ER_ERR_WORKSPACE, "er_csr_from_lens: workspace too small");
  cudaStream_t st = as_stream(stream);
  scan::exclusive_scan(LensIn{lens}, RowPtrOut{row_ptr, n_seg}, n_seg, nullptr, ws, st);
  count_launches(3);
  if (seg_ids && n_lookups_cap > 0) {
    expand_seg_ids_kernel<<<grid_for(n_seg, 256, 8), 256, 0, st>>>(row_ptr, n_seg, n_lookups_cap,
                                                                    seg_ids);
    count_launches(1);
  }
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_bucketize_weighted(const int64_t* ids, const float* weights, const int32_t* seg_ids,
                                     const int32_t* row_ptr, int64_t n_seg, int64_t n_lookups_cap,
                                     const er_slot_t* slots, int32_t n_slots, int64_t* rows,
                                     int32_t* owner, er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(ids && rows && slots, "ids, rows and slots must be non-null");
  ER_REQUIRE(n_slots > 0 && n_slots <= 1024, "n_slots must be in [1, 1024]");
  ER_REQUIRE(n_lookups_cap >= 0 && n_lookups_cap < (1LL << 31), "n_lookups_cap out of range");
  if (n_lookups_cap == 0) return ER_OK;
  cudaStream_t st = as_stream(stream);
  bucketize_kernel<<<grid_for(n_lookups_cap, 256, 8), 256, (size_t)n_slots * sizeof(BucketRule), st>>>(
      ids, weights, seg_ids, row_ptr, n_seg, n_lookups_cap, slots, n_slots, rows, owner);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_bucketize(const int64_t* ids, const int32_t* seg_ids, const int32_t* row_ptr,
                            int64_t n_seg, int64_t n_lookups_cap, const er_slot_t* slots,
                            int32_t n_slots, int64_t* rows, int32_t* owner,
                            er_stream_t stream) {
  return er_bucketize_weighted(ids, nullptr, seg_ids, row_ptr, n_seg, n_lookups_cap, slots, n_slots,
                               rows, owner, stream);
}

extern "C" int er_bucketize_seq(const int64_t* ids, const int32_t* lens, int64_t batch, int32_t seq_len,
                                int32_t n_features, const er_slot_t* slots, int32_t n_slots, int64_t* rows,
                                int32_t* owner, er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(ids && lens && rows && slots, "ids, lens, rows and slots must be non-null");
  ER_REQUIRE(n_slots > 0 && n_slots <= 1024, "n_slots must be in [1, 1024]");
  ER_REQUIRE(batch > 0 && seq_len > 0 && n_features > 0, "batch, seq_len and n_features must be positive");
  const int64_t n_steps = (int64_t)n_features * batch * seq_len;
  ER_REQUIRE(n_steps < (1LL << 31), "n_features * batch * seq_len must fit 31 bits");
  launch_pdl(bucketize_seq_kernel, dim3(grid_for(n_steps, 256, 8)), dim3(256), (size_t)n_slots * sizeof(BucketRule),
             as_stream(stream), ids, lens, n_steps, (int)seq_len, slots, (int)n_slots, rows, owner);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_bucketize_vocab(const int64_t* ids, const float* weights, const int32_t* seg_ids,
                                  const int32_t* row_ptr, int64_t n_seg, int64_t n_lookups_cap,
                                  const er_slot_t* slots, int32_t n_slots, const er_vocab_t* vocabs, int64_t* rows,
                                  int32_t* owner, er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(ids && rows && slots && vocabs, "ids, rows, slots and vocabs must be non-null");
  ER_REQUIRE(n_slots > 0 && n_slots <= 1024, "n_slots must be in [1, 1024]");
  ER_REQUIRE(n_lookups_cap >= 0 && n_lookups_cap < (1LL << 31), "n_lookups_cap out of range");
  if (n_lookups_cap == 0) return ER_OK;
  bucketize_vocab_kernel<false><<<grid_for(n_lookups_cap, 256, 8), 256, (size_t)n_slots * sizeof(BucketRule),
                                  as_stream(stream)>>>(ids, weights, seg_ids, row_ptr, nullptr, n_seg, n_lookups_cap, 1,
                                                       slots, n_slots, vocabs, rows, owner);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_bucketize_seq_vocab(const int64_t* ids, const int32_t* lens, int64_t batch, int32_t seq_len,
                                      int32_t n_features, const er_slot_t* slots, int32_t n_slots,
                                      const er_vocab_t* vocabs, int64_t* rows, int32_t* owner, er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(ids && lens && rows && slots && vocabs, "ids, lens, rows, slots and vocabs must be non-null");
  ER_REQUIRE(n_slots > 0 && n_slots <= 1024, "n_slots must be in [1, 1024]");
  ER_REQUIRE(batch > 0 && seq_len > 0 && n_features > 0, "batch, seq_len and n_features must be positive");
  const int64_t n_steps = (int64_t)n_features * batch * seq_len;
  ER_REQUIRE(n_steps < (1LL << 31), "n_features * batch * seq_len must fit 31 bits");
  launch_pdl(bucketize_vocab_kernel<true>, dim3(grid_for(n_steps, 256, 8)), dim3(256),
             (size_t)n_slots * sizeof(BucketRule), as_stream(stream), ids, (const float*)nullptr,
             (const int32_t*)nullptr, (const int32_t*)nullptr, lens, n_steps, n_steps, (int)seq_len, slots,
             (int)n_slots, vocabs, rows, owner);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}
