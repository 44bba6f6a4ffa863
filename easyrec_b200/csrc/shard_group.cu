// K8: the index-bucketing step of the row-sharded lookup (embedding_parallel_lookup,
// compat/feature_column/feature_column.py:258-303): unique ids, grouped by the rank that owns them, ready for
// the all-to-all.  The reference runs Unique + dynamic_partition and reads the split sizes on the host
// (hvd.alltoall); here the groups have a FIXED capacity per peer, so the three all-to-alls of a step use equal
// splits, nothing is read back and the whole exchange sits inside the step's CUDA graph.
//
//   in : row[l] (owner-local row, -1 = dropped lookup), owner[l] = id mod N          (K1 with shard_n = N)
//   out: send_rows[o * cap + k] = k-th distinct row owned by rank o (rest: -1)
//        pos[l]                 = o * cap + k of lookup l's row (-1 = dropped / over capacity)
//        counts[o]              = distinct rows owned by o (may exceed cap: then counts[N] counts the lost lookups)
//
// Dedup by an open-addressing table in the workspace (keys = row * N + owner, linear probing, 64-bit CAS):
// 2 x n entries of 8 B + 4 B, L2 resident at batch sizes (5 MB at 213K lookups).  Which k a row gets depends on
// the order of the atomics; no result depends on it: the forward reads rows through pos[], the requester sums
// duplicate lookups of a position in lookup order, and the owner sees a row at most once per source rank and sums
// the ranks in rank order (er_embedding_bwd sorts by (row, position) and positions are rank-major).
#include "common.cuh"

namespace er {
namespace sg {

constexpr unsigned long long kEmpty = ~0ull;

__device__ __forceinline__ uint32_t mix(unsigned long long k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdull;
  k ^= k >> 33;
  return (uint32_t)k;
}

struct Args {
  const int64_t* row;
  const int32_t* owner;
  int64_t n;
  int32_t world;
  int64_t cap;
  int64_t* send_rows;
  int64_t* pos;
  int32_t* counts;
  unsigned long long* keys;
  int32_t* vals;
  uint32_t mask;
};

// pass 1: every lookup finds / claims its key's table entry; the claimer takes the next free position of the owner
constexpr int kMaxAgg = 64;   // owners whose position counters a CTA aggregates in shared memory

__global__ void __launch_bounds__(256) insert_kernel(Args a) {
  __shared__ int s_cnt[kMaxAgg], s_base[kMaxAgg];
  const int lane = threadIdx.x & 31;
  const bool agg = a.world <= kMaxAgg;
  if (threadIdx.x < kMaxAgg) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  const int64_t n_pad = (a.n + 255) & ~(int64_t)255;   // whole CTAs run every iteration (block-wide steps below)
  for (int64_t l = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; l < n_pad; l += (int64_t)gridDim.x * blockDim.x) {
    const bool in = l < a.n;
    const int64_t r = in ? a.row[l] : -1;
    const int32_t o = in ? a.owner[l] : -1;
    const bool live = r >= 0 && o >= 0 && o < a.world;
    // (row, owner) -> row * world + owner: one-to-one for every row below 2^63 / world, which covers the 63-bit keys of
    // a key-value table (row = key div N, owner = key mod N) as well as arena rows
    const unsigned long long key = (unsigned long long)r * (unsigned long long)a.world + (unsigned long long)o;
    // lookups of one slot are neighbours and hot ids (one-row tables, the head of a Zipf distribution) repeat
    // thousands of times per batch: one lane per distinct key of the warp talks to the table, the rest copy its answer
    const unsigned peers = __match_any_sync(0xffffffffu, live ? key : (kEmpty - (unsigned)lane));
    const int leader = __ffs(peers) - 1;
    uint32_t h = 0;
    bool won = false;
    if (live && lane == leader) {
      h = mix(key) & a.mask;
      for (;;) {
        unsigned long long old = *reinterpret_cast<volatile unsigned long long*>(a.keys + h);
        if (old == kEmpty) old = atomicCAS(a.keys + h, kEmpty, key);
        if (old == kEmpty) {
          won = true;
          break;
        }
        if (old == key) break;
        h = (h + 1) & a.mask;
      }
    }
    // the claimers take the next free positions of their owners: counted per CTA in shared memory, ONE global
    // atomic per owner and CTA (with two owners, per-claim atomics on two addresses would serialise the kernel)
    int k = 0;
    if (won) k = agg ? atomicAdd(&s_cnt[o], 1) : atomicAdd(a.counts + o, 1);
    if (agg) {
      __syncthreads();
      if ((int)threadIdx.x < a.world) {
        const int c = s_cnt[threadIdx.x];
        s_base[threadIdx.x] = c ? atomicAdd(a.counts + threadIdx.x, c) : 0;
        s_cnt[threadIdx.x] = 0;
      }
      __syncthreads();
      if (won) k += s_base[o];
    }
    if (won) {
      int32_t p = -1;
      if (k < a.cap) {
        p = (int32_t)(o * a.cap + k);
        a.send_rows[p] = r;
      }
      a.vals[h] = p;
    }
    h = __shfl_sync(0xffffffffu, h, leader);
    if (in) a.pos[l] = live ? (int64_t)h : -1;   // resolved to the position by pass 2 (vals[h] may not be written yet)
  }
}

__global__ void __launch_bounds__(256) resolve_kernel(Args a) {
  for (int64_t l = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; l < a.n; l += (int64_t)gridDim.x * blockDim.x) {
    const int64_t h = a.pos[l];
    if (h < 0) continue;
    const int32_t p = a.vals[h];
    if (p < 0) atomicAdd(a.counts + a.world, 1);   // over capacity: the caller checks counts[world]
    a.pos[l] = p;
  }
}

inline uint32_t table_size(int64_t n) {
  uint32_t s = 1024;
  while ((int64_t)s < 2 * n) s <<= 1;
  return s;
}

}  // namespace sg
}  // namespace er

extern "C" size_t er_shard_group_workspace_bytes(int64_t n_lookups) {
  const size_t s = er::sg::table_size(n_lookups > 0 ? n_lookups : 1);
  return s * (sizeof(unsigned long long) + sizeof(int32_t)) + 256;
}

extern "C" int er_shard_group(const int64_t* rows, const int32_t* owner, int64_t n_lookups, int32_t world,
                              int64_t cap_per_peer, int64_t* send_rows, int64_t* pos, int32_t* counts, void* ws,
                              size_t ws_bytes, er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(rows && owner && send_rows && pos && counts, "null argument");
  ER_REQUIRE(n_lookups > 0 && world > 0 && world < 32768 && cap_per_peer > 0, "bad shape");
  ER_REQUIRE((int64_t)world * cap_per_peer < (1ll << 31), "world * cap_per_peer must fit 31 bits");
  if (!ws || ws_bytes < er_shard_group_workspace_bytes(n_lookups))
    return fail(ER_ERR_WORKSPACE, "er_shard_group: workspace too small");
  cudaStream_t st = as_stream(stream);
  sg::Args a;
  a.row = rows;
  a.owner = owner;
  a.n = n_lookups;
  a.world = world;
  a.cap = cap_per_peer;
  a.send_rows = send_rows;
  a.pos = pos;
  a.counts = counts;
  const uint32_t size = sg::table_size(n_lookups);
  a.keys = static_cast<unsigned long long*>(ws);
  a.vals = reinterpret_cast<int32_t*>(a.keys + size);
  a.mask = size - 1;
  cudaMemsetAsync(a.keys, 0xff, (size_t)size * sizeof(unsigned long long), st);
  cudaMemsetAsync(send_rows, 0xff, (size_t)world * cap_per_peer * sizeof(int64_t), st);   // -1
  cudaMemsetAsync(counts, 0, (size_t)(world + 1) * sizeof(int32_t), st);
  const int grid = grid_for(n_lookups, 256, 8);
  sg::insert_kernel<<<grid, 256, 0, st>>>(a);
  sg::resolve_kernel<<<grid, 256, 0, st>>>(a);
  count_launches(2);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}
