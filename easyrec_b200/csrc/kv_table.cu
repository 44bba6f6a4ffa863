// Key-value embedding tables (ev_params): an open-addressing index from 63-bit keys to rows of a preallocated pool.
//
// The reference's counterparts are PAI-TF EmbeddingVariables on one worker and a SOK DynamicVariable under
// EmbeddingParallelStrategy (compat/feature_column/feature_column.py:425-503): a row exists only for a key that has
// been looked up, and two keys never share one.  Here K1 already produces the key (bucket count 2^63 - 1); these kernels
// translate keys into pool rows, and K2 / K7 read and update those rows as any arena row.
//
// Index layout and probe: csrc/kv_index.cuh.  No thread ever waits for another thread's store: the claim launch
// hands each new key a pool row and initialises it, and a second launch reads the row of every lookup's slot.
#include "kv_index.cuh"

namespace er {

constexpr int kKvThreads = 256;

// The initial value of column c of key k's row: a normal(0, stddev), truncated at 2 stddev when `truncated`, drawn by
// inverting the normal CDF at a uniform from a counter-based hash of (seed, key, column).  Independent of insertion
// order, batch order and world size.
__device__ __forceinline__ float kv_init_value(uint64_t seed, int64_t k, int c, float stddev, int truncated) {
  const uint64_t h = kv_mix(seed ^ ((uint64_t)k * 0xD1B54A32D192ED03ull));
  const uint64_t bits = kv_mix(h + (uint64_t)(c + 1) * 0x9E3779B97F4A7C15ull);
  const double u = ((double)(bits >> 11) + 0.5) * 0x1.0p-53;
  // Phi(-2) + u * (Phi(2) - Phi(-2)) for the truncated normal
  const double p = truncated ? 0.022750131948179195 + u * 0.9544997361036416 : u;
  return (float)(normcdfinv(p) * (double)stddev);
}

// the global key of a lookup: a row-sharded table's owner receives key div N and is rank key mod N
__device__ __forceinline__ int64_t kv_global(int64_t k, int shard_n, int shard_rank) {
  return k < 0 ? -1 : k * shard_n + shard_rank;
}

struct KvInit {
  float* weight;
  float* state0;
  float* state1;
  int64_t row_stride;
  int dim;
  float state0_init;
  uint64_t seed;
  float stddev;
  int truncated;
};

__global__ void __launch_bounds__(kKvThreads)
    kv_claim_kernel(KvIndex ix, int64_t capacity, unsigned long long* stats, const int64_t* __restrict__ keys, int64_t n,
                    int shard_n, int shard_rank, int64_t* __restrict__ slots, KvInit in) {
  const int lane = threadIdx.x & 31, t = lane & (kKvTile - 1), base = lane & kKvTile;
  const unsigned tmask = 0xFFFFu << base;
  const int64_t n_tiles = (int64_t)gridDim.x * (blockDim.x / kKvTile);
  for (int64_t l = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / kKvTile; l < n; l += n_tiles) {
    const int64_t k = kv_global(keys[l], shard_n, shard_rank);
    bool won = false;
    const int64_t s = k >= 0 ? kv_probe<true>(ix, k, t, base, tmask, won) : -1;
    if (won) {
      unsigned long long r = 0;
      if (t == 0) r = atomicAdd(stats, 1ull);
      r = __shfl_sync(tmask, r, base);
      const int64_t row = r < (unsigned long long)capacity ? (int64_t)r : -1;
      if (t == 0) ix.rows[s] = row;
      if (row >= 0) {
        const int64_t o = row * in.row_stride;
        for (int c = t; c < in.dim; c += kKvTile) {
          in.weight[o + c] = kv_init_value(in.seed, k, c, in.stddev, in.truncated);
          if (in.state0) in.state0[o + c] = in.state0_init;
          if (in.state1) in.state1[o + c] = 0.f;
        }
      }
    }
    if (t == 0) slots[l] = s;
  }
}

// slots[l] -> the pool row of its key (in place); a live lookup left without a row counts in stats[1]
__global__ void __launch_bounds__(kKvThreads)
    kv_resolve_kernel(const int64_t* __restrict__ index_rows, unsigned long long* stats,
                      const int64_t* __restrict__ keys, int64_t n, int64_t* __restrict__ rows) {
  for (int64_t l = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; l < n; l += (int64_t)gridDim.x * blockDim.x) {
    const int64_t s = rows[l];
    const int64_t r = s >= 0 ? index_rows[s] : -1;
    rows[l] = r;
    if (r < 0 && keys[l] >= 0) atomicAdd(stats + 1, 1ull);
  }
}

__global__ void __launch_bounds__(kKvThreads)
    kv_find_kernel(KvIndex ix, const int64_t* __restrict__ keys, int64_t n, int shard_n, int shard_rank,
                   int64_t zero_row, int64_t* __restrict__ rows) {
  const int lane = threadIdx.x & 31, t = lane & (kKvTile - 1), base = lane & kKvTile;
  const unsigned tmask = 0xFFFFu << base;
  const int64_t n_tiles = (int64_t)gridDim.x * (blockDim.x / kKvTile);
  for (int64_t l = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / kKvTile; l < n; l += n_tiles) {
    const int64_t k = kv_global(keys[l], shard_n, shard_rank);
    bool won;
    const int64_t s = k >= 0 ? kv_probe<false>(ix, k, t, base, tmask, won) : -1;
    const int64_t r = s >= 0 ? ix.rows[s] : -1;
    if (t == 0) rows[l] = k < 0 ? -1 : (r >= 0 ? r : zero_row);
  }
}

__global__ void __launch_bounds__(kKvThreads)
    kv_insert_rows_kernel(KvIndex ix, const int64_t* __restrict__ keys, const int64_t* __restrict__ given, int64_t n,
                          unsigned long long* stats) {
  const int lane = threadIdx.x & 31, t = lane & (kKvTile - 1), base = lane & kKvTile;
  const unsigned tmask = 0xFFFFu << base;
  const int64_t n_tiles = (int64_t)gridDim.x * (blockDim.x / kKvTile);
  for (int64_t l = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / kKvTile; l < n; l += n_tiles) {
    const int64_t k = keys[l];
    bool won = false;
    const int64_t s = k >= 0 ? kv_probe<true>(ix, k, t, base, tmask, won) : -1;
    if (t == 0) {
      if (won)
        ix.rows[s] = given[l];
      else
        atomicAdd(stats + 1, 1ull);   // a negative, repeated or unplaceable key
    }
  }
}

inline int kv_grid(int64_t n, int per_cta) { return grid_for(n, per_cta, 8); }

}  // namespace er

#define ER_KV_REQUIRE_INDEX(keys, rows, n_index)                                                      \
  ER_REQUIRE((keys) && (rows), "null index array");                                                   \
  ER_REQUIRE((n_index) >= 16 && ((n_index) & ((n_index) - 1)) == 0, "n_index must be a power of two >= 16")

extern "C" int er_kv_find_or_insert(int64_t* index_keys, int64_t* index_rows, int64_t n_index, int64_t capacity,
                                    int64_t* stats, const int64_t* keys, int64_t n, int32_t shard_n, int32_t shard_rank,
                                    int64_t* rows, float* weight, float* state0, float* state1, int64_t row_stride,
                                    int32_t dim, float state0_init, uint64_t seed, float init_stddev,
                                    int32_t init_truncated, er_stream_t stream) {
  using namespace er;
  ER_KV_REQUIRE_INDEX(index_keys, index_rows, n_index);
  ER_REQUIRE(stats && weight, "null stats or weight array");
  ER_REQUIRE(n >= 0 && (n == 0 || (keys && rows)), "null keys or rows");
  ER_REQUIRE((const void*)keys != (const void*)rows, "keys and rows must not alias");
  ER_REQUIRE(capacity > 0 && 2 * capacity <= n_index, "n_index must be at least twice the capacity");
  ER_REQUIRE(dim > 0 && row_stride >= dim, "dim must be positive and row_stride >= dim");
  ER_REQUIRE(shard_n > 0 && shard_rank >= 0 && shard_rank < shard_n, "shard_rank must be in [0, shard_n)");
  if (n == 0) return ER_OK;
  const KvIndex ix{(long long*)index_keys, index_rows, n_index / kKvTile};
  const KvInit in{weight, state0, state1, row_stride, dim, state0_init, seed, init_stddev, init_truncated != 0};
  cudaStream_t st = as_stream(stream);
  kv_claim_kernel<<<kv_grid(n, kKvThreads / kKvTile), kKvThreads, 0, st>>>(ix, capacity, (unsigned long long*)stats,
                                                                            keys, n, shard_n, shard_rank, rows, in);
  kv_resolve_kernel<<<kv_grid(n, kKvThreads), kKvThreads, 0, st>>>(index_rows, (unsigned long long*)stats, keys, n,
                                                                   rows);
  count_launches(2);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_kv_find(const int64_t* index_keys, const int64_t* index_rows, int64_t n_index, const int64_t* keys,
                          int64_t n, int32_t shard_n, int32_t shard_rank, int64_t zero_row, int64_t* rows,
                          er_stream_t stream) {
  using namespace er;
  ER_KV_REQUIRE_INDEX(index_keys, index_rows, n_index);
  ER_REQUIRE(shard_n > 0 && shard_rank >= 0 && shard_rank < shard_n, "shard_rank must be in [0, shard_n)");
  ER_REQUIRE(n >= 0 && (n == 0 || (keys && rows)), "null keys or rows");
  if (n == 0) return ER_OK;
  const KvIndex ix{(long long*)index_keys, (int64_t*)index_rows, n_index / kKvTile};
  kv_find_kernel<<<kv_grid(n, kKvThreads / kKvTile), kKvThreads, 0, as_stream(stream)>>>(ix, keys, n, shard_n, shard_rank, zero_row, rows);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_kv_insert_rows(int64_t* index_keys, int64_t* index_rows, int64_t n_index, const int64_t* keys,
                                 const int64_t* rows, int64_t n, int64_t* stats, er_stream_t stream) {
  using namespace er;
  ER_KV_REQUIRE_INDEX(index_keys, index_rows, n_index);
  ER_REQUIRE(stats, "null stats array");
  ER_REQUIRE(n >= 0 && (n == 0 || (keys && rows)), "null keys or rows");
  ER_REQUIRE(2 * n <= n_index, "more keys than half the index");
  if (n == 0) return ER_OK;
  const KvIndex ix{(long long*)index_keys, index_rows, n_index / kKvTile};
  kv_insert_rows_kernel<<<kv_grid(n, kKvThreads / kKvTile), kKvThreads, 0, as_stream(stream)>>>(
      ix, keys, rows, n, (unsigned long long*)stats);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}
