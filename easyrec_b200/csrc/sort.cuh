// Stable LSD radix sort of (row, lookup-position) pairs: the deterministic core
// of the gradient dedup.  It replaces TF's Unique + UnsortedSegmentSum
// (_deduplicate_indexed_slices, applied before compat/adam_s.py:185-213 and
// every TF sparse apply; and array_ops.unique at
// compat/feature_column/feature_column.py:263).
//
// Keys are arena rows (< 2^32 per GPU), values the lookup positions; dropped
// lookups (row < 0) get the sentinel key `n_rows` and sort behind every valid
// row.  8-bit digits, ceil(bits(n_rows)/8) passes (3 for a 10M-row arena).
//
// Shape of the launches: the batch is cut into ~one tile per SM (<= 160 tiles of
// 1024 threads x {2,4,8,16} items), so every launch is a single wave of the 132 SMs.
// P passes -> P + 1 launches, no separate scan kernels:
//   init_hist_kernel : rows -> (key, pos) pairs + per-tile histogram of digit 0;
//                      zeroes the histograms of the later passes
//   scatter_kernel x P: a CTA derives its tile's global offsets by summing the per-tile
//                      histograms over the tiles (4 threads per digit, coalesced column
//                      reads of <= 160 values), ranks its keys stably with warp
//                      match_any, scatters, and counts the NEXT pass's per-tile histogram
//                      at the destination with global atomics (counts are order-free, so
//                      determinism is kept).
// Working set at the benchmark shapes (<= 1M pairs x 8 B x 2 buffers) is L2
// resident (50 MB on the H100): the passes are latency-, not HBM-bound.
#pragma once
#include "common.cuh"

namespace er {
namespace rsort {

constexpr int kRadixBits = 8;
constexpr int kRadix = 1 << kRadixBits;
constexpr int kThreads = 1024;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxPasses = 4;
constexpr int kMaxTiles = 160;

inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// items per thread: smallest of {2, 4, 8, 16} that keeps the tile count <= kMaxTiles
inline int items_for(int64_t n) {
  for (int it = 2; it < 16; it *= 2)
    if (ceil_div(n, (int64_t)kThreads * it) <= kMaxTiles) return it;
  return 16;
}
inline int64_t num_tiles(int64_t n) {
  return n > 0 ? ceil_div(n, (int64_t)kThreads * items_for(n)) : 1;
}

struct Workspace {
  uint32_t* keys_tmp;
  uint32_t* vals_tmp;
  int32_t* hist;  // [kMaxPasses][n_tiles][kRadix]
};

inline size_t workspace_bytes(int64_t n) {
  const int64_t nt = num_tiles(n);
  return align256((size_t)n * 4) * 2 + align256((size_t)kMaxPasses * kRadix * nt * 4) + 512;
}

inline Workspace carve(void* ws, int64_t n) {
  char* p = reinterpret_cast<char*>(align256(reinterpret_cast<size_t>(ws)));
  Workspace w;
  w.keys_tmp = reinterpret_cast<uint32_t*>(p);
  p += align256((size_t)n * 4);
  w.vals_tmp = reinterpret_cast<uint32_t*>(p);
  p += align256((size_t)n * 4);
  w.hist = reinterpret_cast<int32_t*>(p);
  return w;
}

inline int num_passes(int64_t n_rows) {
  int bits = 1;
  while (bits < 32 && (1ULL << bits) <= (uint64_t)n_rows) ++bits;  // sentinel key == n_rows
  return (bits + kRadixBits - 1) / kRadixBits;
}

// One CTA per tile.  zero_me (optional) is cleared by CTA 0 (the backward's hot-row counter).
template <int ITEMS>
static __global__ void __launch_bounds__(kThreads)
    init_hist_kernel(const int64_t* __restrict__ rows, int64_t cap, const int32_t* __restrict__ n_dev,
                     uint32_t sentinel, uint32_t* __restrict__ keys, uint32_t* __restrict__ vals,
                     int32_t* __restrict__ hist, int passes, int32_t* __restrict__ zero_me) {
  __shared__ int s_hist[kRadix];
  const int64_t n_tiles = gridDim.x;
  if (threadIdx.x < kRadix) {
    s_hist[threadIdx.x] = 0;
    for (int p = 1; p < passes; ++p)
      hist[((int64_t)p * n_tiles + blockIdx.x) * kRadix + threadIdx.x] = 0;
  }
  if (zero_me && blockIdx.x == 0 && threadIdx.x < 2) zero_me[threadIdx.x] = 0;  // two counters
  __syncthreads();
  const int64_t n = n_dev ? (int64_t)(*n_dev < cap ? *n_dev : cap) : cap;
  const int64_t base = (int64_t)blockIdx.x * (kThreads * ITEMS);
#pragma unroll
  for (int i = 0; i < ITEMS; ++i) {
    const int64_t idx = base + i * kThreads + threadIdx.x;
    if (idx < cap) {
      const int64_t r = (idx < n) ? rows[idx] : -1;
      const uint32_t k = (r < 0 || r >= (int64_t)sentinel) ? sentinel : (uint32_t)r;
      keys[idx] = k;
      vals[idx] = (uint32_t)idx;
      atomicAdd(&s_hist[k & (kRadix - 1)], 1);
    }
  }
  __syncthreads();
  if (threadIdx.x < kRadix) hist[(int64_t)blockIdx.x * kRadix + threadIdx.x] = s_hist[threadIdx.x];
}

template <int ITEMS>
static __global__ void __launch_bounds__(kThreads)
    scatter_kernel(const uint32_t* __restrict__ keys_in, const uint32_t* __restrict__ vals_in,
                   uint32_t* __restrict__ keys_out, uint32_t* __restrict__ vals_out, int64_t n,
                   int shift, const int32_t* __restrict__ hist_cur, int32_t* __restrict__ hist_next) {
  __shared__ int s_warp_hist[kWarps][kRadix];  // 32 KB
  __shared__ int s_tot[4][kRadix];
  __shared__ int s_bef[4][kRadix];
  __shared__ int s_wsum[kRadix / 32];
  const int n_tiles = gridDim.x;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < kWarps * kRadix; i += kThreads) (&s_warp_hist[0][0])[i] = 0;
  // keys first: their loads overlap the histogram column sums below
  const int64_t base = (int64_t)blockIdx.x * (kThreads * ITEMS) + (int64_t)w * (32 * ITEMS);
  uint32_t key[ITEMS], val[ITEMS];
  int rank[ITEMS];
#pragma unroll
  for (int i = 0; i < ITEMS; ++i) {
    const int64_t idx = base + i * 32 + lane;
    key[i] = (idx < n) ? keys_in[idx] : 0u;
    val[i] = (idx < n) ? vals_in[idx] : 0u;
  }
  // ---- this tile's global offsets: 4 threads per digit each sum a quarter of the tiles ----
  {
    const int d = threadIdx.x & (kRadix - 1), part = threadIdx.x >> kRadixBits;
    const int per = (n_tiles + 3) >> 2;
    const int t0 = part * per, t1 = min(n_tiles, t0 + per);
    int total = 0, before = 0;
    const int32_t* col = hist_cur + d;
    int t = t0;
    for (; t + 8 <= t1; t += 8) {
      int h[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) h[u] = col[(int64_t)(t + u) * kRadix];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        before += (t + u < (int)blockIdx.x) ? h[u] : 0;
        total += h[u];
      }
    }
    for (; t < t1; ++t) {
      const int h = col[(int64_t)t * kRadix];
      before += (t < (int)blockIdx.x) ? h : 0;
      total += h;
    }
    s_tot[part][d] = total;
    s_bef[part][d] = before;
  }
  __syncthreads();
  int digit_base = 0;
  if (threadIdx.x < kRadix) {
    const int d = threadIdx.x;
    const int total = s_tot[0][d] + s_tot[1][d] + s_tot[2][d] + s_tot[3][d];
    const int before = s_bef[0][d] + s_bef[1][d] + s_bef[2][d] + s_bef[3][d];
    // exclusive scan of `total` over the 256 digits (8 warps)
    int incl = total;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (lane == 31) s_wsum[w] = incl;
    digit_base = incl - total + before;
  }
  __syncthreads();
  if (threadIdx.x < kRadix) {
    int off = 0;
    for (int ww = 0; ww < w; ++ww) off += s_wsum[ww];
    digit_base += off;
  }
  // ---- stable rank of every key inside the tile ----
  const unsigned lt_mask = (1u << lane) - 1u;
#pragma unroll
  for (int i = 0; i < ITEMS; ++i) {
    const int64_t idx = base + i * 32 + lane;
    const bool valid = idx < n;
    const int d = (int)((key[i] >> shift) & (kRadix - 1));
    // lanes past the end never match a real digit
    const unsigned peers = __match_any_sync(0xffffffffu, valid ? d : (kRadix + lane));
    const int r = __popc(peers & lt_mask);
    int prev = 0;
    if (valid) prev = s_warp_hist[w][d];
    __syncwarp();
    if (valid && r == 0) s_warp_hist[w][d] = prev + __popc(peers);
    __syncwarp();
    rank[i] = prev + r;
  }
  __syncthreads();
  // ---- local (in-tile) sorted position of every key; delta[d] = global - local offset of digit d ----
  int tile_cnt = 0;
  if (threadIdx.x < kRadix) {
    int run = 0;
#pragma unroll 8
    for (int ww = 0; ww < kWarps; ++ww) {
      int t = s_warp_hist[ww][threadIdx.x];
      s_warp_hist[ww][threadIdx.x] = run;  // entries of this digit in earlier warps of the tile
      run += t;
    }
    tile_cnt = run;
    int incl = tile_cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (lane == 31) s_wsum[w] = incl;
    s_tot[0][threadIdx.x] = incl - tile_cnt;  // exclusive within the warp of digits
  }
  __syncthreads();
  if (threadIdx.x < kRadix) {
    int off = 0;
    for (int ww = 0; ww < w; ++ww) off += s_wsum[ww];
    const int lstart = s_tot[0][threadIdx.x] + off;  // first in-tile slot of this digit
    s_tot[1][threadIdx.x] = lstart;
    s_bef[0][threadIdx.x] = digit_base - lstart;     // delta: global position = local + delta
  }
  __syncthreads();
  // ---- stage the tile in digit order in shared memory, then write runs of equal digits to
  //      consecutive global addresses (coalesced sectors instead of 4-byte scattered stores) ----
  extern __shared__ uint32_t s_stage[];
  uint32_t* s_k = s_stage;
  uint32_t* s_v = s_stage + kThreads * ITEMS;
#pragma unroll
  for (int i = 0; i < ITEMS; ++i) {
    const int64_t idx = base + i * 32 + lane;
    if (idx < n) {
      const int d = (int)((key[i] >> shift) & (kRadix - 1));
      const int lp = s_tot[1][d] + s_warp_hist[w][d] + rank[i];
      s_k[lp] = key[i];
      s_v[lp] = val[i];
    }
  }
  __syncthreads();
  const int64_t tile_base = (int64_t)blockIdx.x * (kThreads * ITEMS);
  const int tile_n = (int)min((int64_t)(kThreads * ITEMS), n - tile_base);
#pragma unroll
  for (int i = 0; i < ITEMS; ++i) {
    const int lp = i * kThreads + threadIdx.x;
    if (lp < tile_n) {
      const uint32_t kk = s_k[lp];
      const int d = (int)((kk >> shift) & (kRadix - 1));
      const int pos = lp + s_bef[0][d];
      keys_out[pos] = kk;
      vals_out[pos] = s_v[lp];
      if (hist_next) {
        const int d2 = (int)((kk >> (shift + kRadixBits)) & (kRadix - 1));
        atomicAdd(&hist_next[(int64_t)(pos / (kThreads * ITEMS)) * kRadix + d2], 1);
      }
    }
  }
}

template <int ITEMS>
inline void sort_rows_t(const int64_t* rows, int64_t cap, const int32_t* n_dev, int64_t n_rows,
                        uint32_t* keys_out, uint32_t* vals_out, void* ws, int32_t* zero_me,
                        cudaStream_t st) {
  Workspace w = carve(ws, cap);
  const int passes = num_passes(n_rows);
  const int64_t nt = num_tiles(cap);
  uint32_t* ka = (passes % 2 == 0) ? keys_out : w.keys_tmp;
  uint32_t* va = (passes % 2 == 0) ? vals_out : w.vals_tmp;
  uint32_t* kb = (passes % 2 == 0) ? w.keys_tmp : keys_out;
  uint32_t* vb = (passes % 2 == 0) ? w.vals_tmp : vals_out;
  // staging buffer of the scatter kernel: (key, val) per tile element; with the 40 KB of static
  // shared memory this exceeds the 48 KB default, so opt in once per instantiation
  constexpr size_t stage_bytes = (size_t)kThreads * ITEMS * 2 * sizeof(uint32_t);
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(scatter_kernel<ITEMS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)stage_bytes);
    attr_set = true;
  }
  init_hist_kernel<ITEMS><<<(unsigned)nt, kThreads, 0, st>>>(rows, cap, n_dev, (uint32_t)n_rows, ka, va,
                                                             w.hist, passes, zero_me);
  for (int p = 0; p < passes; ++p) {
    const int32_t* hc = w.hist + (int64_t)p * nt * kRadix;
    int32_t* hn = (p + 1 < passes) ? w.hist + (int64_t)(p + 1) * nt * kRadix : nullptr;
    scatter_kernel<ITEMS><<<(unsigned)nt, kThreads, stage_bytes, st>>>(ka, va, kb, vb, cap, p * kRadixBits, hc, hn);
    uint32_t* t = ka; ka = kb; kb = t;
    t = va; va = vb; vb = t;
  }
  count_launches(1 + passes);
}

// Sort `cap` pairs; result lands in keys_out / vals_out.
inline void sort_rows(const int64_t* rows, int64_t cap, const int32_t* n_dev, int64_t n_rows,
                      uint32_t* keys_out, uint32_t* vals_out, void* ws, int32_t* zero_me,
                      cudaStream_t st) {
  switch (items_for(cap)) {
    case 2: sort_rows_t<2>(rows, cap, n_dev, n_rows, keys_out, vals_out, ws, zero_me, st); break;
    case 4: sort_rows_t<4>(rows, cap, n_dev, n_rows, keys_out, vals_out, ws, zero_me, st); break;
    case 8: sort_rows_t<8>(rows, cap, n_dev, n_rows, keys_out, vals_out, ws, zero_me, st); break;
    default: sort_rows_t<16>(rows, cap, n_dev, n_rows, keys_out, vals_out, ws, zero_me, st); break;
  }
}

}  // namespace rsort
}  // namespace er
