// K7, bucketed dedup: the (row, lookup) pairs are brought into "equal rows adjacent, ascending lookup order"
// WITHOUT a global sort.
//
//   lookups --multiplicative hash of the row--> NB buckets (two streaming passes over the rows: count, place)
//   one WARP per bucket sorts its pairs in registers on the 64-bit composite (row << 32 | lookup) and writes
//   them out; buckets are laid out back to back, so the result has every run of equal rows contiguous and
//   internally ordered by lookup position - exactly what the run kernels of embedding_bwd.cu need (they never
//   required rows to ascend ACROSS runs).
//
// Against the 3-pass LSD radix sort of sort.cuh (3 x 18 us at the C2 batch, latency bound) this is two cheap
// streaming kernels plus one register-level sort: ~20 us.  A bucket is chosen by a multiplicative hash of the
// row, so clustered ids (identity columns, sequences) spread evenly; only duplicates of one row land together,
// and those are exactly the entries that must meet.  Determinism: placement inside a bucket uses atomics (any
// order), but the in-bucket sort is a total order on (row, lookup position), so the output is unique.
//
// Bucket sizes are exact (pass 1 counts), the pair array is dense.  Size classes:
//   n <= kWarpCap (128)     bk_sort_kernel: one warp, bitonic network over shuffles, 1/2/4 registers per lane
//   n <= kBigCap (16384)    bk_sort_big_kernel: one CTA of 1024 threads, bitonic in 128 KB of shared memory
//   larger                  same kernel, stable LSD radix sort through global memory (slow, correct: needs
//                           > 16K lookups of ONE row in a batch)
// Slots of mode ER_BUCKET_ONE_ROW (a one-row table hit by every sample: RawFeature projections) never enter the
// buckets: their gradient is a weighted column sum (one_row_cta, riding in the sort launch).
#pragma once
#include "common.cuh"
#include "slots.cuh"

namespace er {
namespace bk {

constexpr int kWarpCap = 128;     // pairs a warp sorts in registers (4 per lane)
constexpr int kCap = 1024;        // pairs a 256-thread CTA sorts in shared memory (medium buckets)
constexpr int kThreads = 256;
constexpr int kBigCap = 16384;    // pairs a big-bucket CTA sorts in shared memory (128 KB)
constexpr int kBigThreads = 1024;
constexpr int kCoopRun = 48;      // CTA paths: longer runs are summed by the whole CTA
constexpr int kQueueRun = 4096;   // big buckets: longer runs go to the multi-CTA hot-row kernel
constexpr int kTile = 2048;       // lookups per CTA of the count / place passes
constexpr int kTileThreads = 512;
constexpr int kMaxBuckets = 8192;
constexpr int kOneRowChunk = 512; // samples per CTA of the one-row column sum

// warp mode: about 50-80 lookups per bucket (a warp sorts 64 pairs with two registers per lane);
// CTA mode (rows a warp cannot stage: dim > 32, odd dims): about 200-300 per bucket
inline int num_buckets(int64_t n, bool warp_mode) {
  int nb = 64;
  while (nb < kMaxBuckets && (int64_t)nb * (warp_mode ? 80 : 320) < n) nb <<= 1;
  return nb;
}

__device__ __forceinline__ uint32_t bucket_of(uint32_t key, int log2_nb) {
  return (key * 0x9E3779B1u) >> (32 - log2_nb);
}

struct Ws {
  uint64_t* pairs;      // [n] bucket-ordered (row << 32 | lookup)
  uint64_t* pairs_tmp;  // [n] scratch of the oversized-bucket fallback
  int32_t* bcnt;        // [NB] bucket sizes
  int32_t* bcur;        // [NB] placement cursors
  int32_t* boff;        // [NB + 1] exclusive offsets
  int32_t* big_list;    // [NB] buckets with more than kCap pairs
  int32_t* med_list;    // [NB] buckets with (warp_cap, kCap] pairs
  int32_t* n_big;       // [0] big buckets, [1] medium buckets (+ padding)
};

inline size_t a256(size_t x) { return (x + 255) & ~(size_t)255; }
// The words that must be zero when a call starts lie back to back so that ONE memset clears them:
//   [ bcnt | bcur | n_big ]  (placement state, owned by the call that placed)   zero_place_bytes()
//   [ counters | tickets ]   (hot-row queue + one-row tickets, owned by every K7 call)   zero_call_bytes()
constexpr size_t kCntBytes = ((size_t)(kMaxBuckets + 1) * 4 + 255) & ~(size_t)255;
constexpr size_t kTicketBytes = 2048 * 4;
inline size_t zero_place_bytes() { return 2 * kCntBytes + 256; }
inline size_t zero_call_bytes() { return 256 + kTicketBytes; }
// p: 256-byte aligned.  *counters / *tickets receive the per-call zero block.
inline Ws carve(char* p, int64_t n, int32_t** counters, int32_t** tickets, char** end) {
  Ws w;
  w.pairs = reinterpret_cast<uint64_t*>(p); p += a256((size_t)n * 8);
  w.pairs_tmp = reinterpret_cast<uint64_t*>(p); p += a256((size_t)n * 8);
  w.bcnt = reinterpret_cast<int32_t*>(p); p += kCntBytes;
  w.bcur = reinterpret_cast<int32_t*>(p); p += kCntBytes;
  w.n_big = reinterpret_cast<int32_t*>(p); p += 256;
  *counters = reinterpret_cast<int32_t*>(p); p += 256;
  *tickets = reinterpret_cast<int32_t*>(p); p += kTicketBytes;
  w.boff = reinterpret_cast<int32_t*>(p); p += kCntBytes;
  w.big_list = reinterpret_cast<int32_t*>(p); p += kCntBytes;
  w.med_list = reinterpret_cast<int32_t*>(p); p += kCntBytes;
  *end = p;
  return w;
}

struct PlaceArgs {
  const int64_t* rows;
  int64_t cap;            // lookups (capacity)
  const int32_t* n_dev;   // live lookups (device) or NULL
  uint32_t sentinel;      // n_rows
  const int32_t* seg_ids; // lookup -> segment (NULL: identity)
  const er_slot_t* slots; // to skip ER_BUCKET_ONE_ROW slots (NULL: none)
  int n_slots;
  int log2_nb;
  int warp_cap;           // buckets up to this size are sorted by a warp (0: CTA mode, every bucket is "medium")
  Ws w;
};

// key of lookup l, or the sentinel when it does not take part (dropped, out of range, one-row slot)
__device__ __forceinline__ uint32_t key_of(const PlaceArgs& a, const SlotView& sv, const int* s_one_row, int64_t l,
                                           int64_t n) {
  if (l >= n) return a.sentinel;
  const int64_t r = a.rows[l];
  if (r < 0 || r >= (int64_t)a.sentinel) return a.sentinel;
  if (s_one_row) {
    const int32_t s = a.seg_ids ? a.seg_ids[l] : (int32_t)l;
    if (s_one_row[slot_of(sv, s)]) return a.sentinel;
  }
  return (uint32_t)r;
}

// shared layout of the two placement passes: [slot table | one-row flags (n_slots ints) | counts (NB ints)]
__device__ __forceinline__ int* place_smem(const PlaceArgs& a, unsigned char* s_raw, SlotView* sv, int** one_row) {
  size_t off = 0;
  *one_row = nullptr;
  if (a.slots) {
    *sv = load_slots(s_raw, a.slots, a.n_slots);
    off = (slot_smem_bytes(a.n_slots) + 15) & ~(size_t)15;
    int* f = reinterpret_cast<int*>(s_raw + off);
    int any = 0;
    for (int i = threadIdx.x; i < a.n_slots; i += blockDim.x) {
      f[i] = a.slots[i].bucket_mode == ER_BUCKET_ONE_ROW;
      any |= f[i];
    }
    any = __syncthreads_or(any);
    off += ((size_t)a.n_slots * 4 + 15) & ~(size_t)15;
    if (any) *one_row = f;
  }
  return reinterpret_cast<int*>(s_raw + off);
}
inline size_t place_smem_bytes(int n_slots, int nb, bool with_slots) {
  size_t off = 0;
  if (with_slots) off = ((slot_smem_bytes(n_slots) + 15) & ~(size_t)15) + (((size_t)n_slots * 4 + 15) & ~(size_t)15);
  return off + (size_t)nb * 2 * sizeof(int);
}

// pass 1: bucket sizes
static __global__ void __launch_bounds__(kTileThreads) bk_count_kernel(const __grid_constant__ PlaceArgs a) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  SlotView sv;
  int* one_row;
  int* s_cnt = place_smem(a, s_raw, &sv, &one_row);
  const int nb = 1 << a.log2_nb;
  for (int i = threadIdx.x; i < nb; i += kTileThreads) s_cnt[i] = 0;
  __syncthreads();
  const int64_t n = a.n_dev ? (int64_t)(*a.n_dev < a.cap ? *a.n_dev : a.cap) : a.cap;
  const int64_t base = (int64_t)blockIdx.x * kTile;
#pragma unroll
  for (int i = 0; i < kTile / kTileThreads; ++i) {
    const int64_t l = base + i * kTileThreads + threadIdx.x;
    const uint32_t k = key_of(a, sv, one_row, l, n);
    if (k != a.sentinel) atomicAdd(&s_cnt[bucket_of(k, a.log2_nb)], 1);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nb; i += kTileThreads)
    if (s_cnt[i]) atomicAdd(&a.w.bcnt[i], s_cnt[i]);
}

// pass 2: offsets (every CTA scans the NB counts itself: 4-32 KB out of L2) and placement
static __global__ void __launch_bounds__(kTileThreads) bk_place_kernel(const __grid_constant__ PlaceArgs a) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  __shared__ int s_warp[kTileThreads / 32];
  SlotView sv;
  int* one_row;
  int* s_cnt = place_smem(a, s_raw, &sv, &one_row);
  const int nb = 1 << a.log2_nb;
  int* s_base = s_cnt + nb;
  // exclusive scan of bcnt over the buckets -> s_base
  const int per = (nb + kTileThreads - 1) / kTileThreads;   // consecutive buckets per thread (<= 16)
  int loc[kMaxBuckets / kTileThreads];
  int acc = 0;
#pragma unroll
  for (int u = 0; u < kMaxBuckets / kTileThreads; ++u) {
    const int b = threadIdx.x * per + u;
    loc[u] = (u < per && b < nb) ? a.w.bcnt[b] : 0;
    acc += loc[u];
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int incl = acc;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) s_warp[wid] = incl;
  for (int i = threadIdx.x; i < nb; i += kTileThreads) s_cnt[i] = 0;
  __syncthreads();
  int woff = 0;
  for (int ww = 0; ww < wid; ++ww) woff += s_warp[ww];
  int ex = woff + incl - acc;
#pragma unroll
  for (int u = 0; u < kMaxBuckets / kTileThreads; ++u) {
    const int b = threadIdx.x * per + u;
    if (u < per && b < nb) {
      s_base[b] = ex;
      if (blockIdx.x == 0) {
        a.w.boff[b] = ex;
        if (loc[u] > kCap)
          a.w.big_list[atomicAdd(&a.w.n_big[0], 1)] = b;
        else if (loc[u] > a.warp_cap)
          a.w.med_list[atomicAdd(&a.w.n_big[1], 1)] = b;
      }
      ex += loc[u];
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == kTileThreads - 1) a.w.boff[nb] = ex;
  __syncthreads();
  // local ranks, then one global reservation per touched bucket
  const int64_t n = a.n_dev ? (int64_t)(*a.n_dev < a.cap ? *a.n_dev : a.cap) : a.cap;
  const int64_t base = (int64_t)blockIdx.x * kTile;
  uint32_t key[kTile / kTileThreads];
  int rank[kTile / kTileThreads];
#pragma unroll
  for (int i = 0; i < kTile / kTileThreads; ++i) {
    const int64_t l = base + i * kTileThreads + threadIdx.x;
    key[i] = key_of(a, sv, one_row, l, n);
    rank[i] = 0;
    if (key[i] != a.sentinel) rank[i] = atomicAdd(&s_cnt[bucket_of(key[i], a.log2_nb)], 1);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nb; i += kTileThreads) {
    const int c = s_cnt[i];
    if (c) s_base[i] += atomicAdd(&a.w.bcur[i], c);
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < kTile / kTileThreads; ++i) {
    if (key[i] == a.sentinel) continue;
    const int64_t l = base + i * kTileThreads + threadIdx.x;
    a.w.pairs[s_base[bucket_of(key[i], a.log2_nb)] + rank[i]] = ((uint64_t)key[i] << 32) | (uint32_t)l;
  }
}

// ---- in-CTA pieces -----------------------------------------------------------------------------------
template <int THREADS>
__device__ __forceinline__ void bitonic_sort(uint64_t* s, int P) {
  for (int k = 2; k <= P; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < (P >> 1); t += THREADS) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
        const int l = i | j;
        const uint64_t x = s[i], y = s[l];
        const bool up = (i & k) == 0;
        if ((x > y) == up) {
          s[i] = y;
          s[l] = x;
        }
      }
      __syncthreads();
    }
  }
}

// run starts of the sorted pairs s[0, n): s_start[r] = first index of run r, s_start[R] = n.  Returns R.
// ITEMS consecutive elements per thread (THREADS * ITEMS >= n).
template <int THREADS, int ITEMS, typename IdxT>
__device__ __forceinline__ int run_starts(const uint64_t* s, int n, IdxT* s_start, int* s_warp /*[THREADS/32 + 1]*/) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int i0 = threadIdx.x * ITEMS;
  unsigned heads = 0;
  int cnt = 0;
#pragma unroll
  for (int u = 0; u < ITEMS; ++u) {
    const int i = i0 + u;
    const bool h = i < n && (i == 0 || (uint32_t)(s[i] >> 32) != (uint32_t)(s[i - 1] >> 32));
    heads |= (h ? 1u : 0u) << u;
    cnt += h;
  }
  int incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) s_warp[wid] = incl;
  __syncthreads();
  int woff = 0, total = 0;
  for (int ww = 0; ww < THREADS / 32; ++ww) {
    if (ww < wid) woff += s_warp[ww];
    total += s_warp[ww];
  }
  int r = woff + incl - cnt;
#pragma unroll
  for (int u = 0; u < ITEMS; ++u)
    if ((heads >> u) & 1u) s_start[r++] = (IdxT)(i0 + u);
  if (threadIdx.x == 0) s_start[total] = (IdxT)n;
  __syncthreads();
  return total;
}

}  // namespace bk
}  // namespace er
