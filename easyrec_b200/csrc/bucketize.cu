// K0: lens -> CSR (row_ptr, seg_ids);  K1: raw int64 ids -> arena rows.
//
// Reference ops replaced (SURVEY.md section 2.5 K1):
//   cumsum(lens) + searchsorted        compat/feature_column/feature_column.py:264-266
//   as_string + string_to_hash_bucket_fast   feature_column_v2.py:3915-3921
//   vals % num_buckets                 input/parquet_input.py:221
//   identity column with default 0     feature_column_v2.py:4268-4292
//   uniq % N / int64(recv / N)         compat/feature_column/feature_column.py:296,317
// Both kernels are pure streaming integer work: 8 B in + 8 B out per lookup.
#include "common.cuh"
#include "hash.cuh"
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

__global__ void __launch_bounds__(256)
    bucketize_kernel(const int64_t* __restrict__ ids, const float* __restrict__ weights,
                     const int32_t* __restrict__ seg_ids,
                     const int32_t* __restrict__ row_ptr, int64_t n_seg, int64_t cap,
                     const er_slot_t* __restrict__ slots, int n_slots,
                     int64_t* __restrict__ rows, int32_t* __restrict__ owner) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  BucketRule* tab = reinterpret_cast<BucketRule*>(s_raw);
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
  const int uniform = __syncthreads_and(ok);
  const FastDiv div = make_fastdiv((uint32_t)(nseg0 > 0 ? nseg0 : 1));
  int64_t n = cap;
  if (row_ptr) {
    int64_t t = row_ptr[n_seg];
    n = t < cap ? t : cap;
  }
  for (int64_t l = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; l < n;
       l += (int64_t)gridDim.x * blockDim.x) {
    const int32_t s = seg_ids ? seg_ids[l] : (int32_t)l;
    int f;
    if (uniform) {
      f = (int)fastdiv((uint32_t)s, div);
    } else {
      int lo = 0, hi = n_slots;
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (tab[mid].seg_begin <= s)
          lo = mid;
        else
          hi = mid;
      }
      f = lo;
    }
    const int64_t nb = tab[f].num_buckets;
    const int64_t off = tab[f].row_offset;
    const int mode = tab[f].mode;
    const int shard_n = tab[f].shard_n;
    const int64_t v = ids[l];
    int64_t r;
    bool drop = false;
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
    // _prune_invalid_weights (compat/embedding_ops.py): a mean / sqrtn lookup whose weight is not > 0 (NaN included)
    // is dropped here, so that K2, K7, er_mark_rows and K8 all see it as a dropped lookup
    if (weights && tab[f].combiner != ER_COMBINER_SUM && !(weights[l] > 0.f)) drop = true;
    int32_t own = 0;
    if (shard_n > 1) {
      own = (int32_t)(r % shard_n);
      r = r / shard_n;
    }
    rows[l] = drop ? -1 : (off + r);
    if (owner) owner[l] = drop ? -1 : own;
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
