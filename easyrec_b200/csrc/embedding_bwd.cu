// K7: backward of the gather+pool = gradient dedup + per-row segment sum + fused
// optimizer row update, in one pipeline with no host sync:
//
//   rows[L] --dedup--> (row, lookup) runs: equal rows adjacent, in ascending lookup order
//   G_row = sum over the run, in ascending lookup order, of coef_l * dL/d(pooled[seg(l)])
//   row, state <- optimizer(row, state, G_row * grad_scale)          (same kernel)
//
// Reference ops replaced: the IndexedSlices gradient of embedding_lookup_sparse,
// TF Optimizer._deduplicate_indexed_slices (Unique + UnsortedSegmentSum) and the
// sparse apply: lazy Adam compat/adam_s.py:185-213, TF SparseApplyAdagrad
// (acc += g^2; w -= lr*g*rsqrt(acc); acc0 = 0.1, protos/optimizer.proto:79),
// EP gradient scaling compat/optimizers.py:315-316.
//
// Two dedup engines, chosen by the call:
//  * bucketed (bucket_bwd.cuh + the bk_* kernels below): every table update.  The lookups are hashed into buckets
//    by row (bk_place, which er_embedding_bwd_presort can run ahead), a warp or a CTA sorts each bucket on
//    (row, lookup), and the same kernel sums the runs and applies the optimizer.
//  * radix (sort.cuh + the bwd_runs_* / bwd_scan_* kernels): calls that also emit the deduplicated gradient,
//    compact and sorted by row (uniq_rows / uniq_grads / n_uniq).  P+1 sort launches + a head-rank scan + runs
//    kernel + hot-row kernel.  Dims 64 / 128: a warp scans 32 sorted positions, ballots the run heads and deals
//    them to its dim/4-lane groups, which sum each run in lookup order (the sort is stable); other non-vector
//    dims: a thread per (position, column), in lookup order; dims 4..32 and 1: a lane per lookup and a segmented
//    shuffle scan over the warp (a fixed tree, faster at these widths; last-ulp differences to lookup order).
// Runs longer than kLongRun (radix) or bk::kQueueRun (bucketed) - Zipf-hot ids - are queued as kChunk-lookup work
// items; the hot-row kernel sums one chunk per CTA (one lookup per thread, warp shuffles + a fixed-order
// shared-memory combine), and the CTA that finishes a run last adds the chunk partials in chunk order and applies
// the optimizer: deterministic, no float atomics.
//
// HBM traffic per call (algorithmic): L*8 sorted pairs + L*R gathered upstream gradient
// rows + U*k*R row/state read-modify-write, R = 4*dim, k = 2 (sgd), 4 (adagrad), 6 (adam).
#include "common.cuh"
#include "scan.cuh"
#include "slots.cuh"
#include "sort.cuh"
#include "bucket_bwd.cuh"

namespace er {

struct CBufs {
  const float* p[ER_MAX_BUFS];
};

constexpr int kLongRun = 64;  // runs longer than this go to the chunked CTA-wide kernel
constexpr int kBatch = 4;     // lookups fetched per step of the run loop
constexpr int kChunk = 512;   // lookups per hot-row work item (2 per thread)

struct BwdArgs {
  float* table;
  float* state0;
  float* state1;
  int dim;
  int row_stride;
  uint32_t sentinel;  // == n_rows
  const uint32_t* keys;
  const uint32_t* vals;
  const uint64_t* pairs;  // bucketed engine: sorted (row << 32 | lookup) pairs of the queued hot rows
  int64_t n;  // sorted pairs (== n_lookups_cap)
  const float* weights;
  const int32_t* seg_ids;
  const er_slot_t* slots;
  int n_slots;
  CBufs gbufs;
  const float* seg_scale;
  er_opt_t opt;
  float lr_t;  // adam: lr*sqrt(1-b2^t)/(1-b1^t)
  const float* hyper;  // device float[ER_HYPER_N] overriding opt.lr / beta powers / grad_scale (CUDA graphs)
  int64_t* uniq_rows;
  float* uniq_grads;
  const int32_t* head_rank;  // exclusive count of run heads before each position (emit mode)
  int32_t* counters;         // [0] hot runs, [1] chunks (zeroed by the sort's init kernel)
  int4* long_list;           // per hot run: (start, length, first chunk, n_chunks)
  int32_t* run_done;         // per hot run: chunks finished
  int2* chunk_list;          // per chunk: (run, chunk index)
  float* partials;           // [chunk][dim]
  // one-row slots (ER_BUCKET_ONE_ROW): their column sums are computed by the CTAs behind the first main_ctas of
  // bk_fused_kernel's grid (or_chunks == 0: none)
  const int64_t* or_rows;
  float* or_partials;        // [n_slots][or_chunks][dim]
  int32_t* or_tickets;       // [n_slots], zero between calls
  int or_chunks;
  int main_ctas;
};

// gradient row pointer and coefficient of sorted entry with lookup position l
__device__ __forceinline__ const float* grad_src(const BwdArgs& a, const SlotView& sv, uint32_t l,
                                                 float* coef) {
  const int32_t s = a.seg_ids ? a.seg_ids[l] : (int32_t)l;
  const SlotLite sl = slot_lite(sv, slot_of(sv, s));
  float c = (a.weights && !slot_unit_weights(sl)) ? a.weights[l] : 1.0f;
  if (a.seg_scale) c = __fmul_rn(c, a.seg_scale[s]);
  *coef = c;
  return a.gbufs.p[sl.misc & 0xff] + (int64_t)(s - sl.seg_begin) * sl.out_stride + sl.out_col;
}

struct Hyper {
  float lr, lr_t, grad_scale;
};

// per-step scalars of the row rule: kernel arguments, or - when the caller keeps them in device memory so that a
// captured graph follows a schedule - four broadcast loads by the threads that apply an update
__device__ __forceinline__ Hyper load_hyper(const er_opt_t& o, float lr_t_arg, const float* __restrict__ hyper) {
  Hyper h;
  if (hyper) {
    h.lr = __ldg(hyper + ER_HYPER_LR);
    h.grad_scale = __ldg(hyper + ER_HYPER_GRAD_SCALE);
    h.lr_t = h.lr;
    if (o.kind == ER_OPT_LAZY_ADAM || o.kind == ER_OPT_ADAM_ROWS)
      h.lr_t = adam_lr_t_of(h.lr, __ldg(hyper + ER_HYPER_BETA1_POWER), __ldg(hyper + ER_HYPER_BETA2_POWER));
  } else {
    h.lr = o.lr;
    h.lr_t = lr_t_arg;
    h.grad_scale = o.grad_scale;
  }
  return h;
}

__device__ __forceinline__ void upd_one(const BwdArgs& a, const Hyper& h, float g, float& w, float& s0, float& s1) {
  switch (a.opt.kind) {
    case ER_OPT_ADAGRAD: {
      s0 = __fadd_rn(s0, __fmul_rn(g, g));
      w = __fsub_rn(w, __fmul_rn(__fmul_rn(h.lr, g), __frsqrt_rn(s0)));
      break;
    }
    case ER_OPT_LAZY_ADAM:
    case ER_OPT_ADAM_ROWS: {
      // m_part = g*(1-b1) + m*b1 ; v_part = g*g*(1-b2) + v*b2 ; w += -lr_t*m_part/(sqrt(v_part)+eps)
      s0 = __fadd_rn(__fmul_rn(g, 1.0f - a.opt.beta1), __fmul_rn(s0, a.opt.beta1));
      s1 = __fadd_rn(__fmul_rn(__fmul_rn(g, g), 1.0f - a.opt.beta2), __fmul_rn(s1, a.opt.beta2));
      w = __fadd_rn(w, __fdiv_rn(__fmul_rn(-h.lr_t, s0), __fadd_rn(__fsqrt_rn(s1), a.opt.eps)));
      break;
    }
    case ER_OPT_MOMENTUM: {
      // tf.train.MomentumOptimizer (ApplyMomentum / SparseApplyMomentum, use_nesterov false):
      // accum = accum * momentum + g ; var -= lr * accum   (momentum rides in opt.beta1)
      s0 = __fadd_rn(__fmul_rn(s0, a.opt.beta1), g);
      w = __fsub_rn(w, __fmul_rn(h.lr, s0));
      break;
    }
    default:  // SGD
      w = __fsub_rn(w, __fmul_rn(h.lr, g));
  }
}

__device__ __forceinline__ void f4_fma_sep(float4& g, const float4& v, float c) {
  g.x = __fadd_rn(g.x, __fmul_rn(v.x, c));
  g.y = __fadd_rn(g.y, __fmul_rn(v.y, c));
  g.z = __fadd_rn(g.z, __fmul_rn(v.z, c));
  g.w = __fadd_rn(g.w, __fmul_rn(v.w, c));
}
__device__ __forceinline__ void f4_acc(float4& g, const float4& v) {
  g.x = __fadd_rn(g.x, v.x);
  g.y = __fadd_rn(g.y, v.y);
  g.z = __fadd_rn(g.z, v.z);
  g.w = __fadd_rn(g.w, v.w);
}

__device__ __forceinline__ float4 f4_scale1(const float4& v, float c) {
  return make_float4(__fmul_rn(v.x, c), __fmul_rn(v.y, c), __fmul_rn(v.z, c), __fmul_rn(v.w, c));
}

struct RowRegs {
  float4 w, s0, s1;
};

__device__ __forceinline__ RowRegs load_row(const BwdArgs& a, uint32_t row, int lane) {
  RowRegs r;
  r.w = r.s0 = r.s1 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (!a.table) return r;
  const int64_t off = (int64_t)row * a.row_stride;
  r.w = reinterpret_cast<const float4*>(a.table + off)[lane];
  if (a.state0) r.s0 = reinterpret_cast<const float4*>(a.state0 + off)[lane];
  if (a.state1) r.s1 = reinterpret_cast<const float4*>(a.state1 + off)[lane];
  return r;
}

__device__ __forceinline__ void apply_row_vec(const BwdArgs& a, uint32_t row, int lane, float4 g,
                                              int64_t head_pos, RowRegs r) {
  const Hyper h = load_hyper(a.opt, a.lr_t, a.hyper);
  g.x = __fmul_rn(g.x, h.grad_scale);
  g.y = __fmul_rn(g.y, h.grad_scale);
  g.z = __fmul_rn(g.z, h.grad_scale);
  g.w = __fmul_rn(g.w, h.grad_scale);
  if (a.uniq_rows) {
    const int32_t u = a.head_rank[head_pos];
    if (lane == 0) a.uniq_rows[u] = (int64_t)row;
    reinterpret_cast<float4*>(a.uniq_grads + (int64_t)u * a.dim)[lane] = g;
  }
  if (!a.table) return;
  upd_one(a, h, g.x, r.w.x, r.s0.x, r.s1.x);
  upd_one(a, h, g.y, r.w.y, r.s0.y, r.s1.y);
  upd_one(a, h, g.z, r.w.z, r.s0.z, r.s1.z);
  upd_one(a, h, g.w, r.w.w, r.s0.w, r.s1.w);
  const int64_t off = (int64_t)row * a.row_stride;
  reinterpret_cast<float4*>(a.table + off)[lane] = r.w;
  if (a.state0) reinterpret_cast<float4*>(a.state0 + off)[lane] = r.s0;
  if (a.state1) reinterpret_cast<float4*>(a.state1 + off)[lane] = r.s1;
}

__device__ __forceinline__ void apply_scalar(const BwdArgs& a, uint32_t key, int c, float g,
                                             int64_t head_pos) {
  const Hyper h = load_hyper(a.opt, a.lr_t, a.hyper);
  g = __fmul_rn(g, h.grad_scale);
  if (a.uniq_rows) {
    const int32_t u = a.head_rank[head_pos];
    if (c == 0) a.uniq_rows[u] = (int64_t)key;
    a.uniq_grads[(int64_t)u * a.dim + c] = g;
  }
  if (!a.table) return;
  const int64_t off = (int64_t)key * a.row_stride + c;
  float w = a.table[off];
  float s0 = a.state0 ? a.state0[off] : 0.f;
  float s1 = a.state1 ? a.state1[off] : 0.f;
  upd_one(a, h, g, w, s0, s1);
  a.table[off] = w;
  if (a.state0) a.state0[off] = s0;
  if (a.state1) a.state1[off] = s1;
}

// first index >= lo whose key differs from `key` (keys[lo] == key).  Equal rows are contiguous, but rows need not
// ascend across runs (bucket order), so this gallops forward and bisects on equality, not on order.
__device__ __forceinline__ int64_t run_end(const uint32_t* __restrict__ keys, int64_t lo, int64_t n,
                                           uint32_t key) {
  int64_t step = 1, hi = lo + 1;
  while (hi < n && keys[hi] == key) {
    lo = hi;
    step <<= 1;
    hi = lo + step;
  }
  if (hi > n) hi = n;
  while (hi - lo > 1) {   // keys[lo] == key, keys[hi] != key (or hi == n)
    const int64_t mid = (lo + hi) >> 1;
    if (keys[mid] == key)
      lo = mid;
    else
      hi = mid;
  }
  return hi;
}

// One thread registers a hot run (sorted positions [start, start + len)) and its chunks.
__device__ __forceinline__ void enqueue_run(const BwdArgs& a, int64_t start, int len) {
  const int nch = (len + kChunk - 1) / kChunk;
  const int q = atomicAdd(&a.counters[0], 1);
  const int c0 = atomicAdd(&a.counters[1], nch);
  a.long_list[q] = make_int4((int)start, len, c0, nch);
  a.run_done[q] = 0;
  for (int c = 0; c < nch; ++c) a.chunk_list[c0 + c] = make_int2(q, c);
}

// radix engine: the run of `key` that starts at `start` and still goes on at position j
__device__ __forceinline__ void enqueue_long(const BwdArgs& a, int64_t start, int64_t j, uint32_t key) {
  enqueue_run(a, start, (int)(run_end(a.keys, j, a.n, key) - start));
}

// ---- one-row tables (ER_BUCKET_ONE_ROW slots): weighted column sums -----------------------------------------
// Chunk c of slot f sums coef_b * g[b, cols of f] over its kOneRowChunk samples: lane groups take samples
// g, g + G, ... in order, the groups are added in group order, the chunk partials in chunk order by the slot's
// last CTA, which then applies the optimizer to the row: deterministic.  CTAs of other slots exit at once.
// A slot gets or_chunks CTAs, sized on the average slot; CTA c takes chunks c, c + or_chunks, ... so a slot with
// more segments than that is still covered.  Chunk c's partial sits at f + seg_begin / kOneRowChunk + c: slots are
// disjoint and ordered by seg_begin, so the indices of different slots never meet (and stay below
// max_one_row_parts).
// Their shared memory is declared at namespace scope: the compiler then places it behind bk_fused_kernel's own
// shared variables (s_warp at offset 0), the layout that kernel's code was measured with.
__shared__ __align__(16) float s_or_part[1024];   // vec: G groups x LANES float4; scalar: 256 floats
__shared__ int s_or_last;
__shared__ long long s_or_row;

// every live lookup of a one-row slot names the same row - K1 writes slot.row_offset for all of them, the row-sharded
// exchange (sharded.ShardedLookup) the position of that one row in its send buffer - but any of them may be dropped
// (-1): the row of the first live one, found block by block (all threads of the CTA call this), or -1
__device__ __forceinline__ int64_t one_row_row(const BwdArgs& a, const er_slot_t& sl) {
  for (int base = 0; base < sl.n_seg; base += blockDim.x) {
    const int e = base + threadIdx.x;
    const int64_t r = e < sl.n_seg ? a.or_rows[(int64_t)sl.seg_begin + e] : -1;
    if (threadIdx.x == 0) s_or_row = -1;
    __syncthreads();
    if (r >= 0) s_or_row = r;
    if (__syncthreads_or(r >= 0)) return s_or_row;
  }
  return -1;
}

template <int LANES>
__device__ __forceinline__ void one_row_cta(const BwdArgs& a, int cta) {
  const int f = cta / a.or_chunks, c_first = cta - f * a.or_chunks;
  const er_slot_t sl = a.slots[f];
  if (sl.bucket_mode != ER_BUCKET_ONE_ROW) return;
  constexpr int L = LANES > 0 ? LANES : 1;
  constexpr int G = 256 / L;
  const int dim = a.dim;
  const int used_chunks = (sl.n_seg + bk::kOneRowChunk - 1) / bk::kOneRowChunk;
  if (c_first >= used_chunks) return;
  const int used_ctas = min(a.or_chunks, used_chunks);
  float* const parts = a.or_partials + ((int64_t)f + sl.seg_begin / bk::kOneRowChunk) * dim;   // [chunk][dim]
  const float* gbuf = a.gbufs.p[sl.out_buf];
  if constexpr (LANES > 0) {
    const int grp = threadIdx.x / LANES, lane = threadIdx.x % LANES;
    float4 tot = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int c = c_first; c < used_chunks; c += a.or_chunks) {
      const int s0 = c * bk::kOneRowChunk, s1 = min(sl.n_seg, s0 + bk::kOneRowChunk);
      float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
      constexpr int U = 4;   // samples of a lane group in flight
      for (int e = s0 + grp; e < s1; e += G * U) {
        float4 v[U];
        float coef[U];
        bool use[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int ee = e + u * G;
          use[u] = false;
          if (ee < s1) {
            const int64_t l = (int64_t)sl.seg_begin + ee;   // single-valued slot: lookup == segment
            use[u] = a.or_rows[l] >= 0;                        // a dropped lookup contributes nothing
            coef[u] = a.weights ? a.weights[l] : 1.0f;
            if (a.seg_scale) coef[u] = __fmul_rn(coef[u], a.seg_scale[l]);
            v[u] = reinterpret_cast<const float4*>(gbuf + (int64_t)ee * sl.out_stride + sl.out_col)[lane];
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u)
          if (use[u]) f4_fma_sep(g, v[u], coef[u]);
      }
      reinterpret_cast<float4*>(s_or_part)[grp * LANES + lane] = g;
      __syncthreads();
      tot = make_float4(0.f, 0.f, 0.f, 0.f);
      if (threadIdx.x < LANES) {
        for (int q = 0; q < G; ++q) f4_acc(tot, reinterpret_cast<float4*>(s_or_part)[q * LANES + threadIdx.x]);
        __stcg(reinterpret_cast<float4*>(parts + (int64_t)c * dim) + threadIdx.x, tot);
      }
      __syncthreads();
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_or_last = (atomicAdd(&a.or_tickets[f], 1) == used_ctas - 1);
    __syncthreads();
    if (s_or_last) {
      __threadfence();
      // the chunk partials: fetched in parallel, added in chunk order
      for (int base = 0; base < used_chunks; base += G) {
        const int q = base + grp;
        if (q < used_chunks)
          reinterpret_cast<float4*>(s_or_part)[grp * LANES + lane] =
              __ldcg(reinterpret_cast<const float4*>(parts + (int64_t)q * dim) + lane);
        __syncthreads();
        if (threadIdx.x < LANES) {
          if (base == 0) tot = make_float4(0.f, 0.f, 0.f, 0.f);
          const int m = min(G, used_chunks - base);
          for (int q2 = 0; q2 < m; ++q2) f4_acc(tot, reinterpret_cast<float4*>(s_or_part)[q2 * LANES + threadIdx.x]);
        }
        __syncthreads();
      }
      const int64_t row = one_row_row(a, sl);
      if (threadIdx.x < LANES && row >= 0) {
        RowRegs r = load_row(a, (uint32_t)row, threadIdx.x);
        apply_row_vec(a, (uint32_t)row, threadIdx.x, tot, 0, r);
      }
      if (threadIdx.x == 0) a.or_tickets[f] = 0;
    }
  } else {
    for (int c = c_first; c < used_chunks; c += a.or_chunks) {
      const int s0 = c * bk::kOneRowChunk, s1 = min(sl.n_seg, s0 + bk::kOneRowChunk);
      for (int col = 0; col < dim; ++col) {
        float g = 0.f;
        for (int e = s0 + threadIdx.x; e < s1; e += 256) {
          const int64_t l = (int64_t)sl.seg_begin + e;
          if (a.or_rows[l] < 0) continue;
          float coef = a.weights ? a.weights[l] : 1.0f;
          if (a.seg_scale) coef = __fmul_rn(coef, a.seg_scale[l]);
          g = __fadd_rn(g, __fmul_rn(gbuf[(int64_t)e * sl.out_stride + sl.out_col + col], coef));
        }
        s_or_part[threadIdx.x] = g;
        __syncthreads();
        if (threadIdx.x == 0) {
          float tot = 0.f;
          for (int q = 0; q < 256; ++q) tot = __fadd_rn(tot, s_or_part[q]);
          __stcg(parts + (int64_t)c * dim + col, tot);
        }
        __syncthreads();
      }
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_or_last = (atomicAdd(&a.or_tickets[f], 1) == used_ctas - 1);
    __syncthreads();
    if (s_or_last) {
      __threadfence();
      const int64_t row = one_row_row(a, sl);
      for (int col = threadIdx.x; col < dim && row >= 0; col += 256) {
        float tot = 0.f;
        for (int q = 0; q < used_chunks; ++q) tot = __fadd_rn(tot, __ldcg(parts + (int64_t)q * dim + col));
        apply_scalar(a, (uint32_t)row, col, tot, 0);
      }
    }
    __syncthreads();
    if (s_or_last && threadIdx.x == 0) a.or_tickets[f] = 0;
  }
}

// ---- runs, vector rows (dim = 4*LANES) ---------------------------------------------------
template <int LANES>
__global__ void __launch_bounds__(256) bwd_runs_vec_kernel(const __grid_constant__ BwdArgs a) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  const SlotView sv = load_slots(s_raw, a.slots, a.n_slots);
  constexpr int GROUPS = 32 / LANES;
  const int lane32 = threadIdx.x & 31;
  const int lane = lane32 % LANES;
  const int grp = lane32 / LANES;
  const int64_t base = ((int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 32;
  if (base >= a.n) return;
  const int64_t pos = base + lane32;
  const uint32_t k = pos < a.n ? a.keys[pos] : a.sentinel;
  uint32_t kprev = __shfl_up_sync(0xffffffffu, k, 1);
  if (lane32 == 0) kprev = (base > 0) ? a.keys[base - 1] : ~k;
  const bool is_head = pos < a.n && k < a.sentinel && (pos == 0 || kprev != k);
  const unsigned heads = __ballot_sync(0xffffffffu, is_head);
#pragma unroll 1
  for (int t = 0; t < LANES; ++t) {
    const int p = grp + t * GROUPS;
    if (!((heads >> p) & 1u)) continue;
    const int64_t i = base + p;
    const uint32_t key = a.keys[i];
    RowRegs row = load_row(a, key, lane);  // in flight while the run is summed
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
    int64_t j = i;
    int cnt = 0;
    bool queued = false;
    while (true) {
      uint32_t l[kBatch];
      int m = 0;
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        const bool in = (j + u < a.n);
        const uint32_t kk = in ? a.keys[j + u] : a.sentinel;
        l[u] = in ? a.vals[j + u] : 0u;
        if (m == u && kk == key) m = u + 1;
      }
      float4 gv[kBatch];
      float c[kBatch];
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        if (u < m) {
          const float* src = grad_src(a, sv, l[u], &c[u]);
          gv[u] = reinterpret_cast<const float4*>(src)[lane];
        }
      }
#pragma unroll
      for (int u = 0; u < kBatch; ++u)
        if (u < m) f4_fma_sep(g, gv[u], c[u]);
      j += m;
      cnt += m;
      if (m < kBatch) break;
      if (cnt >= kLongRun) {
        if (j < a.n && a.keys[j] == key) {  // hot row: hand the whole run to the chunked kernel
          if (lane == 0) enqueue_long(a, i, j, key);
          queued = true;
        }
        break;
      }
    }
    if (!queued) apply_row_vec(a, key, lane, g, i, row);
  }
}

// ---- runs, lane-per-lookup segmented scan (dim <= 32) ------------------------------------------
// A warp owns 32 consecutive sorted positions.  Each LANE takes one lookup: it resolves its
// gradient source once (no redundant address math across a lane group) and issues its whole
// 4*LANES-float gradient row at once, so 32 x LANES 16-byte loads are in flight per warp.  Equal
// keys are adjacent, so the per-row sums are a segmented inclusive scan over the lanes (5 shuffle
// steps); the last lane of a segment stages its sum in shared memory and LANES-lane groups then
// apply the optimizer with the row/state loads that were issued before the gradient loads.
// A run that starts in this window and continues past it is finished by this warp (it belongs to
// the warp that holds its head); leading lanes that continue an earlier warp's run are skipped.
// The order of additions is the fixed scan tree (deterministic; differs from sequential order in
// the last ulp).
template <int LANES>
__global__ void __launch_bounds__(256) bwd_scan_vec_kernel(const __grid_constant__ BwdArgs a) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  const SlotView sv = load_slots(s_raw, a.slots, a.n_slots);
  constexpr int D4 = LANES;            // float4 per row
  constexpr int GROUPS = 32 / LANES;
  float4* s_stage = reinterpret_cast<float4*>(s_raw + ((slot_smem_bytes(a.n_slots) + 15) & ~(size_t)15));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float4* my_stage = s_stage + (size_t)warp * 32 * D4;
  __shared__ int s_tail_lane[8][32];
  __shared__ int s_tail_head[8][32];
  const int64_t base = ((int64_t)blockIdx.x * 8 + warp) * 32;
  if (base >= a.n) return;
  const int64_t pos = base + lane;
  const bool in = pos < a.n;
  const uint32_t k = in ? a.keys[pos] : a.sentinel;
  const uint32_t l = in ? a.vals[pos] : 0u;
  const bool valid = in && k < a.sentinel;
  uint32_t kprev = __shfl_up_sync(0xffffffffu, k, 1);
  if (lane == 0) kprev = (base > 0) ? a.keys[base - 1] : ~k;
  uint32_t knext = __shfl_down_sync(0xffffffffu, k, 1);
  if (lane == 31) knext = (base + 32 < a.n) ? a.keys[base + 32] : ~k;
  const bool is_head = valid && (pos == 0 || kprev != k);
  // lanes that continue a run begun in an earlier window are summed by that window's warp
  const uint32_t k0 = __shfl_sync(0xffffffffu, k, 0);
  const int head0 = __shfl_sync(0xffffffffu, (int)is_head, 0);
  const bool owned = valid && (head0 || k != k0);
  bool is_tail = owned && (knext != k);   // lane 31 with a continuing run is fixed up below
  const int cont = __shfl_sync(0xffffffffu, (int)(owned && knext == k), 31);  // last run continues
  const unsigned lt_mask = (1u << lane) - 1u;
  // ---- tails of this window and the row prefetch -------------------------------------------
  const unsigned tails0 = __ballot_sync(0xffffffffu, is_tail || (lane == 31 && cont));
  if (is_tail || (lane == 31 && cont)) s_tail_lane[warp][__popc(tails0 & lt_mask)] = lane;
  __syncwarp();
  const int n_tails = __popc(tails0);
  const int glane = lane % LANES, grp = lane / LANES;
  RowRegs row0, row1;   // the first two rows this lane group will update: loads in flight under the gradient sums
  uint32_t row0_key = a.sentinel, row1_key = a.sentinel;
  if (grp < n_tails) {
    const int tl = s_tail_lane[warp][grp];
    row0_key = a.keys[base + tl];
    row0 = load_row(a, row0_key, glane);
  }
  if (grp + GROUPS < n_tails) {
    const int tl = s_tail_lane[warp][grp + GROUPS];
    row1_key = a.keys[base + tl];
    row1 = load_row(a, row1_key, glane);
  }
  // ---- this lane's gradient row ------------------------------------------------------------
  float4 g[D4];
#pragma unroll
  for (int c = 0; c < D4; ++c) g[c] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (owned) {
    float coef;
    const float4* src = reinterpret_cast<const float4*>(grad_src(a, sv, l, &coef));
    float4 v[D4];
#pragma unroll
    for (int c = 0; c < D4; ++c) v[c] = src[c];
#pragma unroll
    for (int c = 0; c < D4; ++c) f4_fma_sep(g[c], v[c], coef);
  }
  // ---- segmented inclusive scan over equal keys ----------------------------------------------
  int cnt = owned ? 1 : 0;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const uint32_t kk = __shfl_up_sync(0xffffffffu, k, off);
    const int oo = __shfl_up_sync(0xffffffffu, (int)owned, off);
    const int cc = __shfl_up_sync(0xffffffffu, cnt, off);
    const bool take = lane >= off && owned && oo && kk == k;
#pragma unroll
    for (int c = 0; c < D4; ++c) {
      float4 y;
      y.x = __shfl_up_sync(0xffffffffu, g[c].x, off);
      y.y = __shfl_up_sync(0xffffffffu, g[c].y, off);
      y.z = __shfl_up_sync(0xffffffffu, g[c].z, off);
      y.w = __shfl_up_sync(0xffffffffu, g[c].w, off);
      if (take) f4_acc(g[c], y);
    }
    if (take) cnt += cc;
  }
  // ---- a run that leaves the window: finish it here (or hand it to the hot-row kernel) -----------
  int handed_off = 0;
  if (cont) {
    const uint32_t key = __shfl_sync(0xffffffffu, k, 31);
    int total = __shfl_sync(0xffffffffu, cnt, 31);
    const int64_t start = base + 32 - total;
    int64_t j = base + 32;
    while (true) {
      const int64_t p = j + lane;
      const bool m = p < a.n && a.keys[p] == key;
      const unsigned mm = __ballot_sync(0xffffffffu, m);
      float4 x[D4];
#pragma unroll
      for (int c = 0; c < D4; ++c) x[c] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (m) {
        float coef;
        const float4* src = reinterpret_cast<const float4*>(grad_src(a, sv, a.vals[p], &coef));
#pragma unroll
        for (int c = 0; c < D4; ++c) f4_fma_sep(x[c], src[c], coef);
      }
#pragma unroll
      for (int o = 16; o >= 1; o >>= 1) {
#pragma unroll
        for (int c = 0; c < D4; ++c) {
          float4 y;
          y.x = __shfl_xor_sync(0xffffffffu, x[c].x, o);
          y.y = __shfl_xor_sync(0xffffffffu, x[c].y, o);
          y.z = __shfl_xor_sync(0xffffffffu, x[c].z, o);
          y.w = __shfl_xor_sync(0xffffffffu, x[c].w, o);
          f4_acc(x[c], y);
        }
      }
      if (lane == 31) {
#pragma unroll
        for (int c = 0; c < D4; ++c) f4_acc(g[c], x[c]);
      }
      const int got = __popc(mm);
      total += got;
      j += got;
      if (mm != 0xffffffffu) break;
      if (total >= kLongRun) {
        if (j < a.n && a.keys[j] == key) {
          if (lane == 0) enqueue_long(a, start, j, key);
          handed_off = 1;
        }
        break;
      }
    }
  }
  // ---- stage the sums of the runs that END in this warp, then apply -------------------------
  const bool finish = (is_tail || (lane == 31 && cont && !handed_off));
  if (finish) {
#pragma unroll
    for (int c = 0; c < D4; ++c) my_stage[lane * D4 + c] = g[c];
  }
  if (is_tail || (lane == 31 && cont))  // window part of the run length; -1: handed to the hot-row kernel
    s_tail_head[warp][__popc(tails0 & lt_mask)] = (lane == 31 && cont && handed_off) ? -1 : cnt;
  __syncwarp();
  for (int r = grp; r < n_tails; r += GROUPS) {
    const int tl = s_tail_lane[warp][r];
    const int run_cnt = s_tail_head[warp][r];
    if (run_cnt < 0) continue;  // handed to the hot-row kernel
    const uint32_t key = (r == grp) ? row0_key : (r == grp + GROUPS) ? row1_key : a.keys[base + tl];
    RowRegs row = (r == grp) ? row0 : (r == grp + GROUPS) ? row1 : load_row(a, key, glane);
    // head of the run = tail lane - (entries of the run inside this window) + 1; for a run finished
    // by the continuation loop the tail lane is 31 and the count is its window part
    const int64_t head_pos = base + tl - (run_cnt - 1);
    apply_row_vec(a, key, glane, my_stage[tl * D4 + glane], head_pos, row);
  }
}

__device__ __forceinline__ uint32_t key_at(const BwdArgs& a, int64_t i) {
  return a.pairs ? (uint32_t)(a.pairs[i] >> 32) : a.keys[i];
}
__device__ __forceinline__ uint32_t val_at(const BwdArgs& a, int64_t i) {
  return a.pairs ? (uint32_t)a.pairs[i] : a.vals[i];
}

// ---- hot rows, vector: one CTA per chunk of a run; TPE threads share one lookup (TPE = 1 for
// dim <= 32: a thread moves a whole gradient row) -----------------------------------------------
template <int LANES, int TPE>
__global__ void __launch_bounds__(256) bwd_long_vec_kernel(const __grid_constant__ BwdArgs a) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  const SlotView sv = load_slots(s_raw, a.slots, a.n_slots);
  float4* s_part = reinterpret_cast<float4*>(s_raw + ((slot_smem_bytes(a.n_slots) + 15) & ~(size_t)15));
  __shared__ int s_last;
  constexpr int CH = LANES / TPE;  // float4 chunks per thread
  constexpr int G = 256 / TPE;     // lookups in flight per CTA step
  const int lane32 = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int sub = threadIdx.x % TPE;
  const int grp = threadIdx.x / TPE;
  const int n_chunks = a.counters[1];
  for (int x = blockIdx.x; x < n_chunks; x += gridDim.x) {
    const int2 qc = a.chunk_list[x];
    const int4 run = a.long_list[qc.x];
    const int64_t i = run.x;
    const int len = run.y, c0 = run.z, nch = run.w;
    const uint32_t key = key_at(a, i);
    const int e0 = qc.y * kChunk, e1 = min(len, e0 + kChunk);
    float4 g[CH];
#pragma unroll
    for (int c = 0; c < CH; ++c) g[c] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int e = e0 + grp; e < e1; e += 2 * G) {
      const bool two = (e + G < e1);
      float w0, w1 = 0.f;
      const float* p0 = grad_src(a, sv, val_at(a, i + e), &w0);
      const float* p1 = two ? grad_src(a, sv, val_at(a, i + e + G), &w1) : p0;
      float4 v0[CH], v1[CH];
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        v0[c] = reinterpret_cast<const float4*>(p0)[sub * CH + c];
        v1[c] = reinterpret_cast<const float4*>(p1)[sub * CH + c];
      }
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        f4_fma_sep(g[c], v0[c], w0);
        if (two) f4_fma_sep(g[c], v1[c], w1);
      }
    }
    // lanes that hold the same columns: xor-shuffle tree inside the warp ...
#pragma unroll
    for (int o = 16; o >= TPE; o >>= 1) {
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        float4 y;
        y.x = __shfl_xor_sync(0xffffffffu, g[c].x, o);
        y.y = __shfl_xor_sync(0xffffffffu, g[c].y, o);
        y.z = __shfl_xor_sync(0xffffffffu, g[c].z, o);
        y.w = __shfl_xor_sync(0xffffffffu, g[c].w, o);
        f4_acc(g[c], y);
      }
    }
    // ... then the 8 warps in a fixed order through shared memory
    if (lane32 < TPE) {
#pragma unroll
      for (int c = 0; c < CH; ++c) s_part[warp * LANES + lane32 * CH + c] = g[c];
    }
    __syncthreads();
    float4 tot = make_float4(0.f, 0.f, 0.f, 0.f);
    if (threadIdx.x < LANES) {
      for (int ww = 0; ww < 8; ++ww) f4_acc(tot, s_part[ww * LANES + threadIdx.x]);
    }
    bool finish = (nch == 1);
    if (nch > 1) {
      if (threadIdx.x < LANES)
        __stcg(reinterpret_cast<float4*>(a.partials + (int64_t)(c0 + qc.y) * a.dim) + threadIdx.x, tot);
      __threadfence();
      __syncthreads();
      if (threadIdx.x == 0) s_last = (atomicAdd(&a.run_done[qc.x], 1) == nch - 1);
      __syncthreads();
      finish = s_last != 0;
      if (finish && threadIdx.x < LANES) {
        __threadfence();
        tot = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int c = 0; c < nch; ++c)
          f4_acc(tot, __ldcg(reinterpret_cast<const float4*>(a.partials + (int64_t)(c0 + c) * a.dim) +
                             threadIdx.x));
      }
    }
    if (finish && threadIdx.x < LANES) {
      RowRegs row = load_row(a, key, threadIdx.x);
      apply_row_vec(a, key, threadIdx.x, tot, i, row);
    }
    __syncthreads();
  }
}

// ---- scalar rows (wide dim=1 tables, odd dims): one thread per (sorted position, column) ----
__global__ void __launch_bounds__(256) bwd_runs_scalar_kernel(const __grid_constant__ BwdArgs a) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  const SlotView sv = load_slots(s_raw, a.slots, a.n_slots);
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t i = t / a.dim;
  const int c = (int)(t - i * a.dim);
  if (i >= a.n) return;
  const uint32_t key = a.keys[i];
  if (key >= a.sentinel) return;
  if (i > 0 && a.keys[i - 1] == key) return;
  float g = 0.f;
  int64_t j = i;
  for (; j < a.n && a.keys[j] == key; ++j) {
    if (j - i >= kLongRun) {  // hot row
      if (c == 0) enqueue_long(a, i, j, key);
      return;
    }
    float coef;
    const float* src = grad_src(a, sv, a.vals[j], &coef);
    g = __fadd_rn(g, __fmul_rn(src[c], coef));
  }
  apply_scalar(a, key, c, g, i);
}

__global__ void __launch_bounds__(256) bwd_long_scalar_kernel(const __grid_constant__ BwdArgs a) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  const SlotView sv = load_slots(s_raw, a.slots, a.n_slots);
  __shared__ float s_w[8];
  __shared__ int s_last;
  const int lane32 = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n_chunks = a.counters[1];
  for (int x = blockIdx.x; x < n_chunks; x += gridDim.x) {
    const int2 qc = a.chunk_list[x];
    const int4 run = a.long_list[qc.x];
    const int64_t i = run.x;
    const int len = run.y, c0 = run.z, nch = run.w;
    const uint32_t key = key_at(a, i);
    const int e0 = qc.y * kChunk, e1 = min(len, e0 + kChunk);
    for (int c = 0; c < a.dim; ++c) {
      float g = 0.f;
      for (int e = e0 + threadIdx.x; e < e1; e += 256) {
        float coef;
        const float* src = grad_src(a, sv, val_at(a, i + e), &coef);
        g = __fadd_rn(g, __fmul_rn(src[c], coef));
      }
#pragma unroll
      for (int o = 16; o >= 1; o >>= 1) g = __fadd_rn(g, __shfl_xor_sync(0xffffffffu, g, o));
      if (lane32 == 0) s_w[warp] = g;
      __syncthreads();
      if (threadIdx.x == 0) {
        float tot = 0.f;
        for (int ww = 0; ww < 8; ++ww) tot = __fadd_rn(tot, s_w[ww]);
        if (nch == 1)
          apply_scalar(a, key, c, tot, i);
        else
          __stcg(a.partials + (int64_t)(c0 + qc.y) * a.dim + c, tot);
      }
      __syncthreads();
    }
    if (nch > 1) {
      __threadfence();
      __syncthreads();
      if (threadIdx.x == 0) s_last = (atomicAdd(&a.run_done[qc.x], 1) == nch - 1);
      __syncthreads();
      if (s_last) {
        __threadfence();
        for (int col = threadIdx.x; col < a.dim; col += 256) {
          float tot = 0.f;
          for (int c = 0; c < nch; ++c) tot = __fadd_rn(tot, __ldcg(a.partials + (int64_t)(c0 + c) * a.dim + col));
          apply_scalar(a, key, col, tot, i);
        }
      }
      __syncthreads();
    }
  }
}

// ---- dim == 1 (wide tables): lane-per-lookup segmented scan, the run's last lane applies --------
// Same window protocol as bwd_scan_vec_kernel; a "row" is one float (+ its optimizer slots, which the
// interleaved arena keeps in the same 32-byte sector), so every tail lane does its own RMW.
__global__ void __launch_bounds__(256) bwd_scan_d1_kernel(const __grid_constant__ BwdArgs a) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  const SlotView sv = load_slots(s_raw, a.slots, a.n_slots);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t base = ((int64_t)blockIdx.x * 8 + warp) * 32;
  if (base >= a.n) return;
  const int64_t pos = base + lane;
  const bool in = pos < a.n;
  const uint32_t k = in ? a.keys[pos] : a.sentinel;
  const uint32_t l = in ? a.vals[pos] : 0u;
  const bool valid = in && k < a.sentinel;
  uint32_t kprev = __shfl_up_sync(0xffffffffu, k, 1);
  if (lane == 0) kprev = (base > 0) ? a.keys[base - 1] : ~k;
  uint32_t knext = __shfl_down_sync(0xffffffffu, k, 1);
  if (lane == 31) knext = (base + 32 < a.n) ? a.keys[base + 32] : ~k;
  const bool is_head = valid && (pos == 0 || kprev != k);
  const uint32_t k0 = __shfl_sync(0xffffffffu, k, 0);
  const int head0 = __shfl_sync(0xffffffffu, (int)is_head, 0);
  const bool owned = valid && (head0 || k != k0);
  const bool is_tail = owned && (knext != k);
  const int cont = __shfl_sync(0xffffffffu, (int)(owned && knext == k), 31);
  float g = 0.f;
  if (owned) {
    float coef;
    const float* src = grad_src(a, sv, l, &coef);
    g = __fmul_rn(src[0], coef);
  }
  int cnt = owned ? 1 : 0;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const uint32_t kk = __shfl_up_sync(0xffffffffu, k, off);
    const int oo = __shfl_up_sync(0xffffffffu, (int)owned, off);
    const int cc = __shfl_up_sync(0xffffffffu, cnt, off);
    const float y = __shfl_up_sync(0xffffffffu, g, off);
    if (lane >= off && owned && oo && kk == k) {
      g = __fadd_rn(g, y);
      cnt += cc;
    }
  }
  int handed_off = 0;
  if (cont) {
    const uint32_t key = __shfl_sync(0xffffffffu, k, 31);
    int total = __shfl_sync(0xffffffffu, cnt, 31);
    const int64_t start = base + 32 - total;
    int64_t j = base + 32;
    while (true) {
      const int64_t p = j + lane;
      const bool m = p < a.n && a.keys[p] == key;
      const unsigned mm = __ballot_sync(0xffffffffu, m);
      float x = 0.f;
      if (m) {
        float coef;
        const float* src = grad_src(a, sv, a.vals[p], &coef);
        x = __fmul_rn(src[0], coef);
      }
#pragma unroll
      for (int o = 16; o >= 1; o >>= 1) x = __fadd_rn(x, __shfl_xor_sync(0xffffffffu, x, o));
      if (lane == 31) g = __fadd_rn(g, x);
      const int got = __popc(mm);
      total += got;
      j += got;
      if (mm != 0xffffffffu) break;
      if (total >= kLongRun) {
        if (j < a.n && a.keys[j] == key) {
          if (lane == 0) enqueue_long(a, start, j, key);
          handed_off = 1;
        }
        break;
      }
    }
  }
  if (is_tail || (lane == 31 && cont && !handed_off)) apply_scalar(a, k, 0, g, pos - (cnt - 1));
}

// =====================================================================================================
// Bucketed dedup sort (bucket_bwd.cuh): the lookups have been hashed into buckets by row; here every bucket is
// sorted on (row, lookup) and written out, so that the concatenation of the buckets has equal rows adjacent and in
// ascending lookup order - what the run kernels above consume.  One WARP per bucket sorts in registers (bitonic
// network over 32-wide shuffles, no shared memory, no block barriers); the rare bigger buckets go to one CTA each.
// =====================================================================================================
#ifndef ER_BK_MINB
#define ER_BK_MINB 4   // resident CTAs per SM the register allocation of the fused kernel aims for
#endif

struct BkArgs {
  bk::Ws w;
  int log2_nb;
  int warp_ctas;   // CTAs of the warp role (one warp per bucket), 0 in CTA mode
  int med_ctas;    // CTAs of the medium role (they walk med_list)
};

// Sum entries [j0, j1) of the sorted pairs `sp` (shared memory) for one row, sequentially in lookup order.
template <int LANES>
__device__ __forceinline__ float4 sum_entries(const BwdArgs& a, const SlotView& sv, const uint64_t* sp, int j0, int j1,
                                              int lane) {
  float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int j = j0; j < j1; j += kBatch) {
    float4 gv[kBatch];
    float c[kBatch];
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      if (j + u < j1) {
        const float* src = grad_src(a, sv, (uint32_t)sp[j + u], &c[u]);
        gv[u] = reinterpret_cast<const float4*>(src)[lane];
      }
    }
#pragma unroll
    for (int u = 0; u < kBatch; ++u)
      if (j + u < j1) f4_fma_sep(g, gv[u], c[u]);
  }
  return g;
}

constexpr int kStageF4 = 1024;   // float4 slots of the gradient staging buffer (16 KB)
constexpr uint32_t kDonePos = 0xFFFFFFFFu;

template <typename IdxT>
__device__ __forceinline__ bool run_is_long(const IdxT* s_start, int r) {
  return (int)s_start[r + 1] - (int)s_start[r] > bk::kCoopRun;
}

// Runs [0, R) of the sorted window sp[0, s_start[R]).
//  1. runs longer than kCoopRun: the whole CTA sums them straight from global memory with a fixed two-level tree
//     (or, queue_base >= 0 and longer than kQueueRun, hands them to the multi-CTA hot-row kernel - their pairs lie
//     sorted in global memory at queue_base + index); their entries are then marked done;
//  2. everything else in chunks: ALL threads stage the chunk's gradient rows (already multiplied by their
//     coefficients) in shared memory - every load of the chunk is in flight at once, no per-row serial chain - then
//     each lane group walks its runs r = grp, grp + G, ... adding the staged rows in lookup order and applies the
//     optimizer; the next run's table row is requested before the current update is computed.
template <int LANES, int THREADS, typename IdxT>
__device__ __forceinline__ void process_runs_vec(const BwdArgs& a, const SlotView& sv, uint64_t* sp,
                                                 const IdxT* s_start, int R, float4* s_stage, float4* s_part,
                                                 int* s_coop, int* s_ncoop, int64_t queue_base) {
  constexpr int G = THREADS / LANES;
  constexpr int S_ENT = kStageF4 / LANES;
  const int grp = threadIdx.x / LANES, lane = threadIdx.x % LANES;
  if (threadIdx.x == 0) *s_ncoop = 0;
  __syncthreads();
  for (int r = threadIdx.x; r < R; r += THREADS)
    if (run_is_long(s_start, r)) s_coop[atomicAdd(s_ncoop, 1)] = r;
  __syncthreads();
  const int nco = *s_ncoop;
  for (int c = 0; c < nco; ++c) {
    const int r = s_coop[c];
    const int st = s_start[r], en = s_start[r + 1], len = en - st;
    if (queue_base >= 0 && len > bk::kQueueRun) {
      if (threadIdx.x == 0) enqueue_run(a, queue_base + st, len);
    } else {
      // fixed two-level tree: G consecutive sub-ranges summed in lookup order, then added in sub-range order
      const int chunk = (len + G - 1) / G;
      const int j0 = st + grp * chunk, j1 = min(en, j0 + chunk);
      const float4 g = sum_entries<LANES>(a, sv, sp, j0, j1, lane);
      s_part[grp * LANES + lane] = g;
      __syncthreads();
      if (threadIdx.x < LANES) {
        const uint32_t key = (uint32_t)(sp[st] >> 32);
        RowRegs row = load_row(a, key, threadIdx.x);
        const int used = (len + chunk - 1) / chunk;
        float4 tot = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int q = 0; q < used; ++q) f4_acc(tot, s_part[q * LANES + threadIdx.x]);
        apply_row_vec(a, key, threadIdx.x, tot, 0, row);
      }
    }
    __syncthreads();
    for (int i = st + threadIdx.x; i < en; i += THREADS) sp[i] |= (uint64_t)kDonePos;
  }
  __syncthreads();
  // ---- staged chunks ----
  const int n = s_start[R];
  int r = grp;
  while (r < R && run_is_long(s_start, r)) r += G;
  RowRegs row;
  row.w = row.s0 = row.s1 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (r < R) row = load_row(a, (uint32_t)(sp[s_start[r]] >> 32), lane);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int c0 = 0; c0 < n; c0 += S_ENT) {
    const int c1 = min(n, c0 + S_ENT);
    for (int q = threadIdx.x; q < (c1 - c0) * LANES; q += THREADS) {
      const int e = q / LANES;
      const uint32_t pos = (uint32_t)sp[c0 + e];
      if (pos != kDonePos) {
        float coef;
        const float* src = grad_src(a, sv, pos, &coef);
        s_stage[q] = f4_scale1(reinterpret_cast<const float4*>(src)[q % LANES], coef);
      }
    }
    __syncthreads();
    while (r < R && (int)s_start[r] < c1) {
      const int st = s_start[r], en = s_start[r + 1];
      const int lo = max(st, c0), hi = min(en, c1);
      for (int i = lo; i < hi; ++i) f4_acc(acc, s_stage[(i - c0) * LANES + lane]);
      if (en > c1) break;   // the run continues in the next chunk
      const uint32_t key = (uint32_t)(sp[st] >> 32);
      int rn = r + G;
      while (rn < R && run_is_long(s_start, rn)) rn += G;
      RowRegs nxt;
      nxt.w = nxt.s0 = nxt.s1 = make_float4(0.f, 0.f, 0.f, 0.f);
      if (rn < R) nxt = load_row(a, (uint32_t)(sp[s_start[rn]] >> 32), lane);
      apply_row_vec(a, key, lane, acc, 0, row);
      acc = make_float4(0.f, 0.f, 0.f, 0.f);
      row = nxt;
      r = rn;
    }
    __syncthreads();
  }
}

// any dim: one thread per (run, column), same two phases; the staging buffer holds kStageF4 * 4 floats
template <int THREADS, typename IdxT>
__device__ __forceinline__ void process_runs_scalar(const BwdArgs& a, const SlotView& sv, uint64_t* sp,
                                                    const IdxT* s_start, int R, float* s_stagef, float* s_partf,
                                                    int* s_coop, int* s_ncoop, int64_t queue_base) {
  const int dim = a.dim;
  if (threadIdx.x == 0) *s_ncoop = 0;
  __syncthreads();
  for (int r = threadIdx.x; r < R; r += THREADS)
    if (run_is_long(s_start, r)) s_coop[atomicAdd(s_ncoop, 1)] = r;
  __syncthreads();
  const int nco = *s_ncoop;
  for (int cc = 0; cc < nco; ++cc) {
    const int r = s_coop[cc];
    const int st = s_start[r], en = s_start[r + 1], len = en - st;
    if (queue_base >= 0 && len > bk::kQueueRun) {
      if (threadIdx.x == 0) enqueue_run(a, queue_base + st, len);
    } else {
      const int chunk = (len + THREADS - 1) / THREADS;
      const int j0 = st + threadIdx.x * chunk, j1 = min(en, j0 + chunk);
      const int used = (len + chunk - 1) / chunk;
      for (int c = 0; c < dim; ++c) {
        float g = 0.f;
        for (int j = j0; j < j1; ++j) {
          float coef;
          const float* src = grad_src(a, sv, (uint32_t)sp[j], &coef);
          g = __fadd_rn(g, __fmul_rn(src[c], coef));
        }
        s_partf[threadIdx.x] = g;
        __syncthreads();
        if (threadIdx.x == 0) {
          float tot = 0.f;
          for (int q = 0; q < used; ++q) tot = __fadd_rn(tot, s_partf[q]);
          apply_scalar(a, (uint32_t)(sp[st] >> 32), c, tot, 0);
        }
        __syncthreads();
      }
    }
    __syncthreads();
    for (int i = st + threadIdx.x; i < en; i += THREADS) sp[i] |= (uint64_t)kDonePos;
  }
  __syncthreads();
  const int n = s_start[R];
  const int S_ENT = max(1, (kStageF4 * 4) / dim);
  // a thread walks its (run, column) items in order and keeps a run's partial sum across chunks; with more columns
  // than threads two items of one thread could share a run, so the columns go in blocks of THREADS, one pass each
  for (int cb = 0; cb < dim; cb += THREADS) {
    const int width = min(THREADS, dim - cb);
    const int total = R * width;
    int idx = threadIdx.x;
    float acc = 0.f;
    for (int c0 = 0; c0 < n; c0 += S_ENT) {
      const int c1 = min(n, c0 + S_ENT);
      for (int q = threadIdx.x; q < (c1 - c0) * dim; q += THREADS) {
        const int e = q / dim;
        const uint32_t pos = (uint32_t)sp[c0 + e];
        if (pos != kDonePos) {
          float coef;
          const float* src = grad_src(a, sv, pos, &coef);
          s_stagef[q] = __fmul_rn(src[q - e * dim], coef);
        }
      }
      __syncthreads();
      while (idx < total) {
        const int r = idx / width, c = cb + idx - r * width;
        if (run_is_long(s_start, r)) {
          idx += THREADS;
          continue;
        }
        const int st = s_start[r], en = s_start[r + 1];
        if (st >= c1) break;
        const int lo = max(st, c0), hi = min(en, c1);
        for (int i = lo; i < hi; ++i) acc = __fadd_rn(acc, s_stagef[(i - c0) * dim + c]);
        if (en > c1) break;
        apply_scalar(a, (uint32_t)(sp[st] >> 32), c, acc, 0);
        acc = 0.f;
        idx += THREADS;
      }
      __syncthreads();
    }
  }
}

inline size_t bk_reduce_smem(int n_slots, int cap, int threads) {
  return ((slot_smem_bytes(n_slots) + 15) & ~(size_t)15) + (size_t)cap * 8 + (((size_t)(cap + 1) * 2 + 15) & ~(size_t)15) +
         (size_t)max(kStageF4, threads) * 16 + (size_t)(cap / bk::kCoopRun + 2) * 4 + 64;
}

struct BkSmem {
  uint64_t* pairs;
  uint16_t* start;
  float4* stage;
  float4* part;
  int* coop;
  int* ncoop;
};
__device__ __forceinline__ BkSmem bk_carve(unsigned char* s_raw, int n_slots, int cap, int threads) {
  BkSmem m;
  unsigned char* p = s_raw + ((slot_smem_bytes(n_slots) + 15) & ~(size_t)15);
  m.pairs = reinterpret_cast<uint64_t*>(p); p += (size_t)cap * 8;
  m.start = reinterpret_cast<uint16_t*>(p); p += ((size_t)(cap + 1) * 2 + 15) & ~(size_t)15;
  m.stage = reinterpret_cast<float4*>(p); p += (size_t)max(kStageF4, threads) * 16;
  m.part = m.stage;   // the tree partials of the long runs are done with before the staging starts
  m.coop = reinterpret_cast<int*>(p); p += (size_t)(cap / bk::kCoopRun + 1) * 4;
  m.ncoop = reinterpret_cast<int*>(p);
  return m;
}

// compare-exchange of two registers of one lane (indices i < l = i | j of the network)
__device__ __forceinline__ void cx(uint64_t& lo, uint64_t& hi, bool up) {
  if ((lo > hi) == up) {
    const uint64_t t = lo;
    lo = hi;
    hi = t;
  }
}

// ---- warp role: one warp owns a bucket of <= kWarpCap pairs ---------------------------------------------------
// The pairs are sorted in registers (bitonic network over 32-wide shuffles: no shared memory, no block barrier), then
// consumed 32 at a time: all lanes stage the chunk's gradient rows (times their coefficients) in the warp's slice of
// shared memory - every load of the chunk in flight at once - and the 32/LANES lane groups walk the chunk's runs,
// adding the staged rows in lookup order (the order of a sequential CPU segment sum) and applying the optimizer.  A run
// that crosses a chunk boundary hands its partial sum to the next chunk through a carry slot.
template <int LANES>
struct WarpSmem {
  float4 stage[32 * LANES];
  float4 carry[LANES];
  uint32_t keys[32];
};

__device__ __forceinline__ void sort4(uint64_t (&x)[4], int P, int lane) {
  for (int kk = 2; kk <= P; kk <<= 1) {
    for (int j = kk >> 1; j > 0; j >>= 1) {
      if (j == 64) {
        cx(x[0], x[2], ((lane) & kk) == 0);
        cx(x[1], x[3], ((lane + 32) & kk) == 0);
      } else if (j == 32) {
        cx(x[0], x[1], ((lane) & kk) == 0);
        if (P > 64) cx(x[2], x[3], ((lane + 64) & kk) == 0);
      } else {
        const bool lower = (lane & j) == 0;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          if (r * 32 < P) {
            const uint64_t other = __shfl_xor_sync(0xffffffffu, x[r], j);
            const bool up = ((lane + 32 * r) & kk) == 0;
            // this lane keeps the smaller of the pair iff it holds the lower index of an ascending pair (or the
            // higher index of a descending one): one 64-bit compare, one select
            if ((x[r] > other) == (lower == up)) x[r] = other;
          }
        }
      }
    }
  }
}

template <int LANES>
__device__ __forceinline__ void warp_bucket_vec(const BwdArgs& a, const SlotView& sv, const BkArgs& k, int b,
                                                WarpSmem<LANES>* ws) {
  constexpr int G = 32 / LANES;
  const int lane = threadIdx.x & 31;
  const int gi = lane / LANES, gl = lane % LANES;
  const int n = k.w.bcnt[b];
  if (n == 0 || n > bk::kWarpCap) return;   // empty, or a bucket of the medium / big CTAs
  const int64_t off = k.w.boff[b];
  uint64_t x[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int q = r * 32 + lane;
    x[r] = q < n ? k.w.pairs[off + q] : ~0ull;
  }
  sort4(x, n <= 32 ? 32 : (n <= 64 ? 64 : 128), lane);
  uint32_t carry_key = 0xFFFFFFFFu;   // no run is open
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    if (r * 32 >= n) break;
    const uint32_t key = (uint32_t)(x[r] >> 32), pos = (uint32_t)x[r];
    const int nv = min(32, n - r * 32);   // valid lanes are a prefix
    const uint32_t next_first = (r < 3 && (r + 1) * 32 < n) ? __shfl_sync(0xffffffffu, (uint32_t)(x[r < 3 ? r + 1 : 3] >> 32), 0)
                                                            : 0xFFFFFFFFu;
    uint32_t prevk = __shfl_up_sync(0xffffffffu, key, 1);
    if (lane == 0) prevk = carry_key;
    const bool is_head = lane < nv && key != prevk;
    const unsigned H = __ballot_sync(0xffffffffu, is_head);
    const int nh = __popc(H);
    ws->keys[lane] = key;
    const float4 open_sum = ws->carry[gl];   // read before this chunk may overwrite it (ordered by the __syncwarp below)
    // the table rows of this group's first two runs: requested first, they arrive under the gradient staging
    RowRegs row0, row1;
    row0.w = row0.s0 = row0.s1 = row1.w = row1.s0 = row1.s1 = make_float4(0.f, 0.f, 0.f, 0.f);
    {
      const unsigned h0 = __fns(H, 0, gi + 1), h1 = __fns(H, 0, gi + G + 1);
      const uint32_t k0 = __shfl_sync(0xffffffffu, key, h0 & 31), k1 = __shfl_sync(0xffffffffu, key, h1 & 31);
      if (gi < nh) row0 = load_row(a, k0, gl);
      if (gi + G < nh) row1 = load_row(a, k1, gl);
    }
    // stage the chunk: LANES lanes fetch one gradient row, G rows per step
#pragma unroll
    for (int t = 0; t < LANES; ++t) {
      const int e = t * G + gi;
      const uint32_t pe = __shfl_sync(0xffffffffu, pos, e);
      if (e < nv) {
        float coef;
        const float* src = grad_src(a, sv, pe, &coef);
        ws->stage[e * LANES + gl] = f4_scale1(reinterpret_cast<const float4*>(src)[gl], coef);
      }
    }
    __syncwarp();
    const uint32_t lastk = ws->keys[31];
    const bool chunk_open = (nv == 32) && next_first == lastk;   // the chunk's last run goes on in the next chunk
    // the entries in front of the first head continue the run the previous chunk left open
    const int lead = nh ? (__ffs(H) - 1) : nv;
    if (lead > 0 && gi == 0) {
      float4 acc = open_sum;
      for (int i = 0; i < lead; ++i) f4_acc(acc, ws->stage[i * LANES + gl]);
      if (lead == 32 && chunk_open) {
        ws->carry[gl] = acc;
      } else {
        RowRegs row = load_row(a, carry_key, gl);
        apply_row_vec(a, carry_key, gl, acc, 0, row);
      }
    }
    for (int q = gi; q < nh; q += G) {
      const int h = __fns(H, 0, q + 1);
      const unsigned rest = (h == 31) ? 0u : (H >> (h + 1)) << (h + 1);
      const int e_end = rest ? (__ffs(rest) - 1) : nv;
      const uint32_t kh = ws->keys[h];
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int i = h; i < e_end; ++i) f4_acc(acc, ws->stage[i * LANES + gl]);
      if (e_end == 32 && chunk_open) {
        ws->carry[gl] = acc;
      } else {
        RowRegs row = (q == gi) ? row0 : (q == gi + G) ? row1 : load_row(a, kh, gl);
        apply_row_vec(a, kh, gl, acc, 0, row);
      }
    }
    carry_key = chunk_open ? lastk : 0xFFFFFFFFu;
    __syncwarp();
  }
}

// scalar rows - dim 1 (wide tables), and the warp-placed dims whose operands are not 16-byte aligned: a lane per run,
// the staged values are single floats, one pass over the sorted chunks per column
struct WarpSmem1 {
  float stage[32];
  float carry;
  uint32_t keys[32];
};

__device__ __forceinline__ void warp_bucket_scalar(const BwdArgs& a, const SlotView& sv, const BkArgs& k, int b,
                                                   WarpSmem1* ws) {
  const int lane = threadIdx.x & 31;
  const int n = k.w.bcnt[b];
  if (n == 0 || n > bk::kWarpCap) return;
  const int64_t off = k.w.boff[b];
  uint64_t x[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int q = r * 32 + lane;
    x[r] = q < n ? k.w.pairs[off + q] : ~0ull;
  }
  sort4(x, n <= 32 ? 32 : (n <= 64 ? 64 : 128), lane);
#pragma unroll 1
  for (int col = 0; col < a.dim; ++col) {
    uint32_t carry_key = 0xFFFFFFFFu;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      if (r * 32 >= n) break;
      const uint32_t key = (uint32_t)(x[r] >> 32), pos = (uint32_t)x[r];
      const int nv = min(32, n - r * 32);
      const uint32_t next_first = (r < 3 && (r + 1) * 32 < n) ? __shfl_sync(0xffffffffu, (uint32_t)(x[r < 3 ? r + 1 : 3] >> 32), 0)
                                                              : 0xFFFFFFFFu;
      uint32_t prevk = __shfl_up_sync(0xffffffffu, key, 1);
      if (lane == 0) prevk = carry_key;
      const bool is_head = lane < nv && key != prevk;
      const unsigned H = __ballot_sync(0xffffffffu, is_head);
      const int nh = __popc(H);
      ws->keys[lane] = key;
      const float open_sum = ws->carry;   // read before this chunk may overwrite it
      if (lane < nv) {
        float coef;
        const float* src = grad_src(a, sv, pos, &coef);
        ws->stage[lane] = __fmul_rn(src[col], coef);
      }
      __syncwarp();
      const uint32_t lastk = ws->keys[31];
      const bool chunk_open = (nv == 32) && next_first == lastk;
      const int lead = nh ? (__ffs(H) - 1) : nv;
      if (lead > 0 && lane == 31) {   // (lane 31 never owns a head run of its own beyond the 32nd: see below)
        float acc = open_sum;
        for (int i = 0; i < lead; ++i) acc = __fadd_rn(acc, ws->stage[i]);
        if (lead == 32 && chunk_open)
          ws->carry = acc;
        else
          apply_scalar(a, carry_key, col, acc, 0);
      }
      if (lane < nh && !(lead > 0 && lane == 31)) {
        const int h = __fns(H, 0, lane + 1);
        const unsigned rest = (h == 31) ? 0u : (H >> (h + 1)) << (h + 1);
        const int e_end = rest ? (__ffs(rest) - 1) : nv;
        float acc = 0.f;
        for (int i = h; i < e_end; ++i) acc = __fadd_rn(acc, ws->stage[i]);
        if (e_end == 32 && chunk_open)
          ws->carry = acc;
        else
          apply_scalar(a, ws->keys[h], col, acc, 0);
      }
      carry_key = chunk_open ? lastk : 0xFFFFFFFFu;
      __syncwarp();
    }
  }
}

constexpr bool warp_mode_lanes(int lanes) { return lanes == 1 || lanes == 2 || lanes == 4 || lanes == 8; }

template <int LANES>
inline size_t bk_fused_smem(int n_slots, bool warp_mode) {
  size_t warp_bytes = 0;
  if (warp_mode) {
    if constexpr (LANES > 0)
      warp_bytes = ((slot_smem_bytes(n_slots) + 15) & ~(size_t)15) + 8 * sizeof(WarpSmem<(LANES > 0 && LANES <= 8) ? LANES : 1>);
    else
      warp_bytes = ((slot_smem_bytes(n_slots) + 15) & ~(size_t)15) + 8 * sizeof(WarpSmem1);
  }
  const size_t med = bk_reduce_smem(n_slots, bk::kCap, bk::kThreads);
  return warp_bytes > med ? warp_bytes : med;
}

// One launch, three roles by block index:
//   [0, warp_ctas)                       8 warps, one bucket each (vector rows up to dim 32, and dim 1)
//   [warp_ctas, warp_ctas + med_ctas)    a CTA sorts a medium bucket (warp_cap < n <= kCap) in shared memory
//   behind them                          column sums of the one-row slots
template <int LANES>
__global__ void __launch_bounds__(bk::kThreads, ER_BK_MINB) bk_fused_kernel(const __grid_constant__ BwdArgs a,
                                                                const __grid_constant__ BkArgs k) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  __shared__ int s_warp[bk::kThreads / 32 + 1];
  // (block order = scheduling order; measured at C2: the many short warp CTAs first, the few long-running ones -
  //  hot medium buckets, one-row column sums - behind them is ~15% faster than the other way round)
  const int bid = blockIdx.x;
  if (bid >= k.warp_ctas + k.med_ctas) {
    one_row_cta<LANES>(a, bid - k.warp_ctas - k.med_ctas);
    return;
  }
  const SlotView sv = load_slots(s_raw, a.slots, a.n_slots);
  if (bid < k.warp_ctas) {
    unsigned char* p = s_raw + ((slot_smem_bytes(a.n_slots) + 15) & ~(size_t)15);
    const int b = bid * 8 + (threadIdx.x >> 5);
    if constexpr (LANES > 0 && LANES <= 8) {
      warp_bucket_vec<LANES>(a, sv, k, b, reinterpret_cast<WarpSmem<LANES>*>(p) + (threadIdx.x >> 5));
    } else if constexpr (LANES == 0) {
      warp_bucket_scalar(a, sv, k, b, reinterpret_cast<WarpSmem1*>(p) + (threadIdx.x >> 5));
    }
    return;
  }
  const BkSmem m = bk_carve(s_raw, a.n_slots, bk::kCap, bk::kThreads);
  const int n_med = k.w.n_big[1];
  for (int xi = bid - k.warp_ctas; xi < n_med; xi += k.med_ctas) {
    const int b = k.w.med_list[xi];
    const int n = k.w.bcnt[b];
    const int off = k.w.boff[b];
    int P = 32;
    while (P < n) P <<= 1;
    for (int i = threadIdx.x; i < P; i += bk::kThreads) m.pairs[i] = i < n ? k.w.pairs[off + i] : ~0ull;
    __syncthreads();
    bk::bitonic_sort<bk::kThreads>(m.pairs, P);
    const int R = bk::run_starts<bk::kThreads, bk::kCap / bk::kThreads>(m.pairs, n, m.start, s_warp);
    if constexpr (LANES > 0)
      process_runs_vec<LANES, bk::kThreads>(a, sv, m.pairs, m.start, R, m.stage, m.part, m.coop, m.ncoop, -1);
    else
      process_runs_scalar<bk::kThreads>(a, sv, m.pairs, m.start, R, reinterpret_cast<float*>(m.stage),
                                        reinterpret_cast<float*>(m.part), m.coop, m.ncoop, -1);
    __syncthreads();
  }
}

// One pass of a CTA-local stable LSD radix sort through global memory (oversized buckets only).
// Returns false (and moves nothing) when every element has the same digit.
__device__ __forceinline__ bool cta_radix_pass(const uint64_t* __restrict__ in, uint64_t* __restrict__ out, int n,
                                               int shift, int* s_wh /*[32][256]*/, int* s_cur /*[256]*/) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;
  for (int i = threadIdx.x; i < 256; i += bk::kBigThreads) s_cur[i] = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += bk::kBigThreads) atomicAdd(&s_cur[(int)((in[i] >> shift) & 255)], 1);
  __syncthreads();
  int single = 0;
  if (threadIdx.x < 256) single = (s_cur[threadIdx.x] == n);
  if (__syncthreads_or(single)) return false;
  if (threadIdx.x < 32) {   // exclusive scan of the 256 digit counts
    int carry = 0;
    for (int base = 0; base < 256; base += 32) {
      const int v = s_cur[base + lane];
      int incl = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      s_cur[base + lane] = carry + incl - v;
      carry += __shfl_sync(0xffffffffu, incl, 31);
    }
  }
  __syncthreads();
  for (int base = 0; base < n; base += bk::kBigThreads) {
    for (int i = threadIdx.x; i < 32 * 256; i += bk::kBigThreads) s_wh[i] = 0;
    __syncthreads();
    const int i = base + threadIdx.x;
    const bool valid = i < n;
    const uint64_t e = valid ? in[i] : 0ull;
    const int d = (int)((e >> shift) & 255);
    const unsigned peers = __match_any_sync(0xffffffffu, valid ? d : (256 + lane));
    const int r = __popc(peers & lt_mask);
    if (valid && r == 0) s_wh[wid * 256 + d] = __popc(peers);
    __syncthreads();
    if (threadIdx.x < 256) {
      int run = s_cur[threadIdx.x];
      for (int ww = 0; ww < 32; ++ww) {
        const int t = s_wh[ww * 256 + threadIdx.x];
        s_wh[ww * 256 + threadIdx.x] = run;
        run += t;
      }
      s_cur[threadIdx.x] = run;
    }
    __syncthreads();
    if (valid) out[s_wh[wid * 256 + d] + r] = e;
    __syncthreads();
  }
  return true;
}

// big buckets: a few CTAs (one per SM, kBigCap pairs of shared memory) walk the list of buckets above kCap
template <int LANES>
__global__ void __launch_bounds__(bk::kBigThreads) bk_reduce_big_kernel(const __grid_constant__ BwdArgs a,
                                                                        const __grid_constant__ BkArgs k) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  __shared__ int s_warp[bk::kBigThreads / 32 + 1];
  __shared__ int s_flag;
  const int n_big = k.w.n_big[0];
  if ((int)blockIdx.x >= n_big) return;
  const SlotView sv = load_slots(s_raw, a.slots, a.n_slots);
  const BkSmem m = bk_carve(s_raw, a.n_slots, bk::kBigCap, bk::kBigThreads);
  for (int x = blockIdx.x; x < n_big; x += gridDim.x) {
    const int b = k.w.big_list[x];
    const int n = k.w.bcnt[b];
    const int64_t off = k.w.boff[b];
    uint64_t* gp = k.w.pairs + off;
    bool sorted_in_global = false;
    if (n > bk::kBigCap) {
      // more than kBigCap lookups in one bucket (>= thousands of duplicates of one row): stable LSD radix sort of the
      // 64-bit composites through global memory, digits that do not vary are skipped
      int* s_wh = reinterpret_cast<int*>(m.pairs);
      int* s_cur = s_wh + 32 * 256;
      uint64_t* src = gp;
      uint64_t* dst = k.w.pairs_tmp + off;
      for (int shift = 0; shift < 64; shift += 8) {
        if (cta_radix_pass(src, dst, n, shift, s_wh, s_cur)) {
          uint64_t* t = src; src = dst; dst = t;
        }
        __syncthreads();
      }
      if (src != gp) {
        for (int i = threadIdx.x; i < n; i += bk::kBigThreads) gp[i] = src[i];
      }
      __threadfence_block();
      __syncthreads();
      sorted_in_global = true;
    }
    int p = 0;
    while (p < n) {
      const int mwin = min(bk::kBigCap, n - p);
      if (!sorted_in_global) {
        int P = 32;
        while (P < mwin) P <<= 1;
        for (int i = threadIdx.x; i < P; i += bk::kBigThreads) m.pairs[i] = i < mwin ? gp[i] : ~0ull;
        __syncthreads();
        bk::bitonic_sort<bk::kBigThreads>(m.pairs, P);
      } else {
        for (int i = threadIdx.x; i < mwin; i += bk::kBigThreads) m.pairs[i] = gp[p + i];
        __syncthreads();
      }
      int R = bk::run_starts<bk::kBigThreads, bk::kBigCap / bk::kBigThreads>(m.pairs, mwin, m.start, s_warp);
      int advance = mwin;
      if (sorted_in_global && p + mwin < n &&
          (uint32_t)(m.pairs[mwin - 1] >> 32) == (uint32_t)(gp[p + mwin] >> 32)) {
        // the last run of the window continues past it
        if (R == 1) {   // the window is one run: find its end, queue it (len > kBigCap > kQueueRun)
          const uint32_t key = (uint32_t)(m.pairs[0] >> 32);
          int lo = p + mwin, hi = n;
          while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if ((uint32_t)(gp[mid] >> 32) <= key) lo = mid + 1; else hi = mid;
          }
          if (threadIdx.x == 0) enqueue_run(a, off + p, lo - p);
          p = lo;
          __syncthreads();
          continue;
        }
        advance = m.start[R - 1];
        R -= 1;
      }
      // does any run of this window go to the hot-row kernel?  then its pairs must lie sorted in global memory
      if (!sorted_in_global) {
        if (threadIdx.x == 0) s_flag = 0;
        __syncthreads();
        for (int r = threadIdx.x; r < R; r += bk::kBigThreads)
          if (m.start[r + 1] - m.start[r] > bk::kQueueRun) s_flag = 1;
        __syncthreads();
        if (s_flag)
          for (int i = threadIdx.x; i < mwin; i += bk::kBigThreads) gp[i] = m.pairs[i];
      }
      if constexpr (LANES > 0)
        process_runs_vec<LANES, bk::kBigThreads>(a, sv, m.pairs, m.start, R, m.stage, m.part, m.coop, m.ncoop, off + p);
      else
        process_runs_scalar<bk::kBigThreads>(a, sv, m.pairs, m.start, R, reinterpret_cast<float*>(m.stage),
                                             reinterpret_cast<float*>(m.part), m.coop, m.ncoop, off + p);
      p += advance;
      __syncthreads();
    }
  }
}

struct HeadIn {
  const uint32_t* keys;
  uint32_t sentinel;
  __device__ int operator()(int64_t j) const {
    uint32_t k = keys[j];
    return (k < sentinel && (j == 0 || keys[j - 1] != k)) ? 1 : 0;
  }
};
struct HeadOut {
  int32_t* rank;
  __device__ void operator()(int64_t j, int ex, int) const { rank[j] = ex; }
};

inline size_t a256(size_t x) { return (x + 255) & ~(size_t)255; }

struct BwdWs {
  uint32_t* keys;
  uint32_t* vals;
  int32_t* head_rank;
  int4* long_list;
  int32_t* run_done;
  int2* chunk_list;
  float* partials;
  int32_t* counters;
  void* sort_ws;
  void* scan_ws;
  bk::Ws bk;          // bucketed dedup (bucket_bwd.cuh)
  int32_t* tickets;   // one-row slots: CTAs finished per slot
  float* one_row_partials;
};

inline int64_t max_long_runs(int64_t n) { return n / kLongRun + 1; }
inline int64_t max_chunks(int64_t n) { return n / kChunk + max_long_runs(n) + 1; }
inline int64_t max_one_row_parts(int64_t n) { return n / bk::kOneRowChunk + 2048 + 1; }

// The workspace layout: parts carved from `ws` aligned up to 256 bytes; *end receives the end of the last part.
inline BwdWs bwd_carve(void* ws, int64_t n, int dim, char** end = nullptr) {
  char* p = reinterpret_cast<char*>(a256(reinterpret_cast<size_t>(ws)));
  BwdWs w;
  w.keys = reinterpret_cast<uint32_t*>(p); p += a256((size_t)n * 4);
  w.vals = reinterpret_cast<uint32_t*>(p); p += a256((size_t)n * 4);
  w.head_rank = reinterpret_cast<int32_t*>(p); p += a256((size_t)n * 4);
  w.long_list = reinterpret_cast<int4*>(p); p += a256((size_t)max_long_runs(n) * 16);
  w.run_done = reinterpret_cast<int32_t*>(p); p += a256((size_t)max_long_runs(n) * 4);
  w.chunk_list = reinterpret_cast<int2*>(p); p += a256((size_t)max_chunks(n) * 8);
  w.partials = reinterpret_cast<float*>(p); p += a256((size_t)max_chunks(n) * dim * 4);
  w.bk = bk::carve(p, n, &w.counters, &w.tickets, &p);
  w.one_row_partials = reinterpret_cast<float*>(p); p += a256((size_t)max_one_row_parts(n) * dim * 4);
  w.sort_ws = p; p += a256(rsort::workspace_bytes(n));
  w.scan_ws = p; p += a256(scan::workspace_bytes(n));
  if (end) *end = p;
  return w;
}

// the layout carved from a null base, plus 768 bytes of slack (aligning the caller's base takes at most 255)
inline size_t bwd_ws_bytes(int64_t n, int dim) {
  char* end;
  bwd_carve(nullptr, n, dim, &end);
  return reinterpret_cast<size_t>(end) + 768;
}

static float adam_lr_t(const er_opt_t& o) { return adam_lr_t_of(o.lr, o.beta1_power, o.beta2_power); }

// the hot-row kernel of both engines: sums the queued runs chunk by chunk and applies them
template <int LANES>
static void launch_long(const BwdArgs& a, cudaStream_t st) {
  const size_t sl = slot_smem_bytes(a.n_slots);
  if constexpr (LANES > 0) {
    constexpr int TPE = (LANES <= 8) ? 1 : LANES;
    const size_t smem_long = ((sl + 15) & ~(size_t)15) + (size_t)8 * LANES * sizeof(float4);
    bwd_long_vec_kernel<LANES, TPE><<<4 * kSmCount, 256, smem_long, st>>>(a);
  } else {
    bwd_long_scalar_kernel<<<4 * kSmCount, 256, sl, st>>>(a);
  }
}

// radix engine: runs kernel, then the hot-row kernel.  Vector rows and dim 1: a warp per 32 sorted positions,
// 8 warps per CTA; other dims: a thread per (sorted position, column).
template <int LANES>
static void launch_radix(const BwdArgs& a, cudaStream_t st) {
  const size_t smem = slot_smem_bytes(a.n_slots);
  const unsigned grid = (unsigned)ceil_div(a.n, 256);
  if constexpr (LANES > 8) {
    bwd_runs_vec_kernel<LANES><<<grid, 256, smem, st>>>(a);
  } else if constexpr (LANES > 0) {
    const size_t smem_scan = ((smem + 15) & ~(size_t)15) + (size_t)8 * 32 * LANES * sizeof(float4);
    bwd_scan_vec_kernel<LANES><<<grid, 256, smem_scan, st>>>(a);
  } else if (a.dim == 1) {
    bwd_scan_d1_kernel<<<grid, 256, smem, st>>>(a);
  } else {
    bwd_runs_scalar_kernel<<<(unsigned)ceil_div(a.n * a.dim, 256), 256, smem, st>>>(a);
  }
  launch_long<LANES>(a, st);
  count_launches(2);
}

// ---- bucketed path: host side ------------------------------------------------------------------------------
static int log2_of(int v) {
  int l = 0;
  while ((1 << l) < v) ++l;
  return l;
}

// zero the placement state, count, place.  one_row: slots of mode ER_BUCKET_ONE_ROW are left out.
// rows a warp can stage (vector rows up to dim 32, and the wide dim-1 tables) use one warp per small bucket
static bool k7_warp_mode(int dim) { return dim == 1 || dim == 4 || dim == 8 || dim == 16 || dim == 32; }

static void bk_place(const int64_t* rows, int64_t cap, const int32_t* n_dev, int64_t n_rows, const int32_t* seg_ids,
                     const er_slot_t* slots, int n_slots, bool one_row, bool warp_mode, const BwdWs& w,
                     bool zero_call_block, cudaStream_t st) {
  bk::PlaceArgs pa;
  pa.rows = rows;
  pa.cap = cap;
  pa.n_dev = n_dev;
  pa.sentinel = (uint32_t)n_rows;
  pa.seg_ids = seg_ids;
  pa.slots = one_row ? slots : nullptr;
  pa.n_slots = n_slots;
  const int nb = bk::num_buckets(cap, warp_mode);
  pa.log2_nb = log2_of(nb);
  pa.warp_cap = warp_mode ? bk::kWarpCap : 0;
  pa.w = w.bk;
  cudaMemsetAsync(w.bk.bcnt, 0, bk::zero_place_bytes() + (zero_call_block ? bk::zero_call_bytes() : 0), st);
  const size_t smem = bk::place_smem_bytes(n_slots, nb, pa.slots != nullptr);
  static bool attr = false;
  if (!attr) {
    const int mx = (int)bk::place_smem_bytes(2048, bk::kMaxBuckets, true);
    cudaFuncSetAttribute(bk::bk_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, mx);
    cudaFuncSetAttribute(bk::bk_place_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, mx);
    attr = true;
  }
  const unsigned tiles = (unsigned)ceil_div(cap, (int64_t)bk::kTile);
  bk::bk_count_kernel<<<tiles, bk::kTileThreads, smem, st>>>(pa);
  bk::bk_place_kernel<<<tiles, bk::kTileThreads, smem, st>>>(pa);
  count_launches(2);
}

// per-bucket sort + sums + row update over a placement (bk_place) made in `place_warp_mode`
template <int LANES>
static void bk_launch_fused(BwdArgs a, const BwdWs& place, bool place_warp_mode, cudaStream_t st) {
  BkArgs k;
  k.w = place.bk;
  const int nb = bk::num_buckets(a.n, place_warp_mode);
  k.log2_nb = log2_of(nb);
  k.warp_ctas = place_warp_mode ? (nb >> 3) : 0;
  k.med_ctas = place_warp_mode ? kSmCount : nb;
  const size_t smem = bk_fused_smem<LANES>(a.n_slots, place_warp_mode);
  const size_t smem_big = bk_reduce_smem(a.n_slots, bk::kBigCap, bk::kBigThreads);
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(bk_fused_kernel<LANES>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)bk_fused_smem<LANES>(2048, true));
    cudaFuncSetAttribute(bk_fused_kernel<LANES>, cudaFuncAttributePreferredSharedMemoryCarveout,
                         (int)cudaSharedmemCarveoutMaxShared);
    cudaFuncSetAttribute(bk_reduce_big_kernel<LANES>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)bk_reduce_smem(2048, bk::kBigCap, bk::kBigThreads));
    attr = true;
  }
  const int extra = a.or_chunks * a.n_slots;
  a.main_ctas = k.warp_ctas + k.med_ctas;
  bk_fused_kernel<LANES><<<k.warp_ctas + k.med_ctas + extra, bk::kThreads, smem, st>>>(a, k);
  bk_reduce_big_kernel<LANES><<<kSmCount, bk::kBigThreads, smem_big, st>>>(a, k);
  launch_long<LANES>(a, st);
  count_launches(3);
}

}  // namespace er

extern "C" size_t er_sort_workspace_bytes(int64_t n) { return er::rsort::workspace_bytes(n > 0 ? n : 1); }

extern "C" int er_sort_rows(const int64_t* rows, int64_t n, const int32_t* n_dev, int64_t max_row,
                            uint32_t* keys_out, uint32_t* vals_out, void* ws, size_t ws_bytes,
                            er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(rows && keys_out && vals_out, "null argument");
  ER_REQUIRE(n > 0 && n < (1LL << 31), "n out of range");
  ER_REQUIRE(max_row > 0 && max_row < 0xFFFFFFFFLL, "max_row must be in (0, 2^32-1)");
  if (!ws || ws_bytes < rsort::workspace_bytes(n))
    return fail(ER_ERR_WORKSPACE, "er_sort_rows: workspace too small");
  rsort::sort_rows(rows, n, n_dev, max_row, keys_out, vals_out, ws, nullptr, as_stream(stream));
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" size_t er_embedding_bwd_workspace_bytes(int64_t n_lookups_cap, int32_t dim) {
  return er::bwd_ws_bytes(n_lookups_cap > 0 ? n_lookups_cap : 1, dim > 0 ? dim : 1);
}

static int embedding_bwd_impl(float* table, float* state0, float* state1, int64_t n_rows,
                              int32_t dim, int32_t row_stride, const int64_t* rows,
                              const float* weights, const int32_t* seg_ids,
                              const int32_t* row_ptr, int64_t n_seg, int64_t n_lookups_cap,
                              const er_slot_t* slots, int32_t n_slots,
                              const float* const* grad_bufs, int32_t n_bufs,
                              const float* seg_scale, const er_opt_t* opt, int64_t* uniq_rows,
                              float* uniq_grads, int32_t* n_uniq, void* ws, size_t ws_bytes,
                              const void* sorted_ws, size_t sorted_ws_bytes, int32_t sorted_dim,
                              er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(rows && slots && grad_bufs && opt, "null argument");
  ER_REQUIRE(table || uniq_rows, "nothing to do: table and uniq_rows are both NULL");
  ER_REQUIRE((uniq_rows == nullptr) == (uniq_grads == nullptr) &&
                 (uniq_rows == nullptr) == (n_uniq == nullptr),
             "uniq_rows, uniq_grads and n_uniq go together");
  ER_REQUIRE(dim > 0 && row_stride >= dim, "bad dim / row_stride");
  // the CTA roles stage at least one whole gradient row in their kStageF4 * 4 floats of shared memory
  ER_REQUIRE(dim <= kStageF4 * 4, "dim must be at most 4096");
  ER_REQUIRE(n_rows > 0 && n_rows < 0xFFFFFFFFLL, "n_rows must be in (0, 2^32-1)");
  ER_REQUIRE(n_slots > 0 && n_slots <= 2048, "n_slots must be in [1, 2048]");
  ER_REQUIRE(n_bufs > 0 && n_bufs <= ER_MAX_BUFS, "n_bufs must be in [1, ER_MAX_BUFS]");
  ER_REQUIRE(n_lookups_cap >= 0 && n_lookups_cap < (1LL << 31), "n_lookups_cap out of range");
  ER_REQUIRE(row_ptr || seg_ids || n_lookups_cap == n_seg,
             "without row_ptr / seg_ids every segment must hold exactly one lookup");
  ER_REQUIRE(!row_ptr || seg_ids, "CSR input needs seg_ids (er_csr_from_lens)");
  if (table) {
    const int k = opt->kind;
    ER_REQUIRE(k == ER_OPT_SGD || k == ER_OPT_ADAGRAD || k == ER_OPT_LAZY_ADAM || k == ER_OPT_ADAM_ROWS || k == ER_OPT_MOMENTUM,
               "unknown optimizer kind");
    ER_REQUIRE(k == ER_OPT_SGD || state0, "optimizer state0 missing");
    ER_REQUIRE((k != ER_OPT_LAZY_ADAM && k != ER_OPT_ADAM_ROWS) || state1, "adam needs state1 (v)");
  }
  if (n_lookups_cap == 0) return ER_OK;
  if (!ws || ws_bytes < bwd_ws_bytes(n_lookups_cap, dim))
    return fail(ER_ERR_WORKSPACE, "er_embedding_bwd: workspace too small");
  cudaStream_t st = as_stream(stream);
  BwdWs w = bwd_carve(ws, n_lookups_cap, dim);
  // number of live lookups: row_ptr[n_seg] when CSR (device side), else the capacity
  const int32_t* n_dev = row_ptr ? row_ptr + n_seg : nullptr;
  // Two dedup engines.  Bucketed (bucket_bwd.cuh) updates tables; the global radix sort + scan serves the calls that
  // also want the deduplicated gradient written out sorted by row (uniq_rows).
  const bool bucketed = (uniq_rows == nullptr);
  // one-row slots (ER_BUCKET_ONE_ROW) bypass the dedup when lookup == segment (no CSR lookups in the call)
  const bool one_row = bucketed && seg_ids == nullptr;
  BwdWs src = w;
  if (sorted_ws) {
    // the same lookups were placed / sorted by an earlier call on this stream (a table with the same row plan)
    if (sorted_ws_bytes < bwd_ws_bytes(n_lookups_cap, sorted_dim))
      return fail(ER_ERR_WORKSPACE, "er_embedding_bwd_reuse_sort: source workspace too small");
    if (!bucketed)
      return fail(ER_ERR_UNSUPPORTED, "er_embedding_bwd_reuse_sort: uniq_rows output needs the rows (er_embedding_bwd)");
    if (k7_warp_mode(sorted_dim) != k7_warp_mode(dim))
      return fail(ER_ERR_UNSUPPORTED, "er_embedding_bwd_reuse_sort: the placement was made in the other placement mode "
                                      "(warp-sized buckets for dims 1, 4, 8, 16 and 32, CTA-sized for the others)");
    src = bwd_carve(const_cast<void*>(sorted_ws), n_lookups_cap, sorted_dim);
    cudaMemsetAsync(w.counters, 0, bk::zero_call_bytes(), st);
  } else if (bucketed) {
    bk_place(rows, n_lookups_cap, n_dev, n_rows, seg_ids, slots, n_slots, one_row, k7_warp_mode(dim), w, true, st);
  } else {
    rsort::sort_rows(rows, n_lookups_cap, n_dev, n_rows, w.keys, w.vals, w.sort_ws, w.counters, st);
  }
  const bool place_warp = k7_warp_mode(dim);

  BwdArgs a = {};
  a.table = table;
  a.state0 = state0;
  a.state1 = state1;
  a.dim = dim;
  a.row_stride = row_stride;
  a.sentinel = (uint32_t)n_rows;
  a.keys = w.keys;
  a.vals = w.vals;
  a.pairs = nullptr;
  a.n = n_lookups_cap;
  a.weights = weights;
  a.seg_ids = seg_ids;
  a.slots = slots;
  a.n_slots = n_slots;
  bool aligned = true;
  for (int i = 0; i < ER_MAX_BUFS; ++i) {
    a.gbufs.p[i] = i < n_bufs ? grad_bufs[i] : nullptr;
    if (i < n_bufs) {
      ER_REQUIRE(grad_bufs[i] != nullptr, "null gradient buffer");
      aligned = aligned && (reinterpret_cast<uintptr_t>(grad_bufs[i]) % 16 == 0);
    }
  }
  a.seg_scale = seg_scale;
  a.opt = *opt;
  a.lr_t = (opt->kind == ER_OPT_LAZY_ADAM || opt->kind == ER_OPT_ADAM_ROWS) ? adam_lr_t(*opt) : opt->lr;
  a.hyper = opt->hyper_dev;
  a.uniq_rows = uniq_rows;
  a.uniq_grads = uniq_grads;
  a.head_rank = nullptr;
  a.counters = w.counters;
  a.long_list = w.long_list;
  a.run_done = w.run_done;
  a.chunk_list = w.chunk_list;
  a.partials = w.partials;
  a.or_rows = rows;
  a.or_partials = w.one_row_partials;
  a.or_tickets = w.tickets;
  // CTAs per one-row slot: enough for the average slot (a longer one is strided over, see one_row_cta)
  a.or_chunks = one_row ? (int)ceil_div(ceil_div(n_lookups_cap, (int64_t)n_slots), (int64_t)bk::kOneRowChunk) : 0;
  if (uniq_rows) {
    scan::exclusive_scan(HeadIn{w.keys, a.sentinel}, HeadOut{w.head_rank}, n_lookups_cap, n_uniq,
                         w.scan_ws, st);
    a.head_rank = w.head_rank;
    count_launches(3);
  }
  if (table) {
    aligned = aligned && reinterpret_cast<uintptr_t>(table) % 16 == 0 && row_stride % 4 == 0 &&
              (!state0 || reinterpret_cast<uintptr_t>(state0) % 16 == 0) &&
              (!state1 || reinterpret_cast<uintptr_t>(state1) % 16 == 0);
  }
  if (uniq_grads) aligned = aligned && reinterpret_cast<uintptr_t>(uniq_grads) % 16 == 0;
  const bool vec_dim = (dim == 4 || dim == 8 || dim == 16 || dim == 32 || dim == 64 || dim == 128);
  if (bucketed) {
    ER_REQUIRE(table != nullptr, "the bucketed path updates a table");
    a.keys = nullptr;
    a.vals = nullptr;
    a.pairs = src.bk.pairs;
    if (vec_dim && aligned) {
      switch (dim / 4) {
        case 1: bk_launch_fused<1>(a, src, place_warp, st); break;
        case 2: bk_launch_fused<2>(a, src, place_warp, st); break;
        case 4: bk_launch_fused<4>(a, src, place_warp, st); break;
        case 8: bk_launch_fused<8>(a, src, place_warp, st); break;
        case 16: bk_launch_fused<16>(a, src, place_warp, st); break;
        default: bk_launch_fused<32>(a, src, place_warp, st); break;
      }
    } else {
      bk_launch_fused<0>(a, src, place_warp, st);
    }
    ER_CUDA_LAUNCH_CHECK();
    return ER_OK;
  }
  if (vec_dim && aligned) {
    switch (dim / 4) {
      case 1: launch_radix<1>(a, st); break;
      case 2: launch_radix<2>(a, st); break;
      case 4: launch_radix<4>(a, st); break;
      case 8: launch_radix<8>(a, st); break;
      case 16: launch_radix<16>(a, st); break;
      default: launch_radix<32>(a, st); break;
    }
  } else {
    launch_radix<0>(a, st);
  }
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_embedding_bwd(float* table, float* state0, float* state1, int64_t n_rows,
                                int32_t dim, int32_t row_stride, const int64_t* rows,
                                const float* weights, const int32_t* seg_ids,
                                const int32_t* row_ptr, int64_t n_seg, int64_t n_lookups_cap,
                                const er_slot_t* slots, int32_t n_slots,
                                const float* const* grad_bufs, int32_t n_bufs,
                                const float* seg_scale, const er_opt_t* opt, int64_t* uniq_rows,
                                float* uniq_grads, int32_t* n_uniq, void* ws, size_t ws_bytes,
                                er_stream_t stream) {
  return embedding_bwd_impl(table, state0, state1, n_rows, dim, row_stride, rows, weights, seg_ids, row_ptr,
                            n_seg, n_lookups_cap, slots, n_slots, grad_bufs, n_bufs, seg_scale, opt,
                            uniq_rows, uniq_grads, n_uniq, ws, ws_bytes, nullptr, 0, 0, stream);
}

extern "C" int er_embedding_bwd_presort(const int64_t* rows, int64_t n_rows, const int32_t* seg_ids,
                                        const int32_t* row_ptr, int64_t n_seg, int64_t n_lookups_cap,
                                        const er_slot_t* slots, int32_t n_slots, int32_t dim, void* ws,
                                        size_t ws_bytes, er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(rows && slots, "null argument");
  ER_REQUIRE(n_rows > 0 && n_rows < 0xFFFFFFFFLL, "n_rows must be in (0, 2^32-1)");
  ER_REQUIRE(n_slots > 0 && n_slots <= 2048, "n_slots must be in [1, 2048]");
  ER_REQUIRE(n_lookups_cap >= 0 && n_lookups_cap < (1LL << 31) && dim > 0, "bad shape");
  if (n_lookups_cap == 0) return ER_OK;
  if (!ws || ws_bytes < bwd_ws_bytes(n_lookups_cap, dim))
    return fail(ER_ERR_WORKSPACE, "er_embedding_bwd_presort: workspace too small");
  BwdWs w = bwd_carve(ws, n_lookups_cap, dim);
  const int32_t* n_dev = row_ptr ? row_ptr + n_seg : nullptr;
  bk_place(rows, n_lookups_cap, n_dev, n_rows, seg_ids, slots, n_slots, seg_ids == nullptr, k7_warp_mode(dim), w, false,
           as_stream(stream));
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_embedding_bwd_reuse_sort(float* table, float* state0, float* state1, int64_t n_rows,
                                           int32_t dim, int32_t row_stride, const int64_t* rows,
                                           const float* weights, const int32_t* seg_ids,
                                           const int32_t* row_ptr, int64_t n_seg, int64_t n_lookups_cap,
                                           const er_slot_t* slots, int32_t n_slots,
                                           const float* const* grad_bufs, int32_t n_bufs,
                                           const float* seg_scale, const er_opt_t* opt, int64_t* uniq_rows,
                                           float* uniq_grads, int32_t* n_uniq, void* ws, size_t ws_bytes,
                                           const void* sorted_ws, size_t sorted_ws_bytes,
                                           int32_t sorted_dim, er_stream_t stream) {
  if (!sorted_ws) return er::fail(ER_ERR_INVALID_ARG, "er_embedding_bwd_reuse_sort: sorted_ws is NULL");
  if (!rows) return er::fail(ER_ERR_INVALID_ARG, "er_embedding_bwd_reuse_sort: rows is NULL");
  return embedding_bwd_impl(table, state0, state1, n_rows, dim, row_stride, rows, weights, seg_ids,
                            row_ptr, n_seg, n_lookups_cap, slots, n_slots, grad_bufs, n_bufs, seg_scale,
                            opt, uniq_rows, uniq_grads, n_uniq, ws, ws_bytes, sorted_ws, sorted_ws_bytes,
                            sorted_dim, stream);
}

namespace er {

__global__ void __launch_bounds__(256)
    sparse_apply_kernel(const __grid_constant__ BwdArgs a, const int64_t* __restrict__ uniq_rows,
                        const float* __restrict__ uniq_grads, const int32_t* __restrict__ n_uniq,
                        int64_t n_cap) {
  const int64_t n = n_uniq ? (int64_t)(*n_uniq < n_cap ? *n_uniq : n_cap) : n_cap;
  const Hyper h = load_hyper(a.opt, a.lr_t, a.hyper);
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n * a.dim;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t u = t / a.dim;
    const int c = (int)(t - u * a.dim);
    const int64_t row = uniq_rows[u];
    if (row < 0) continue;
    const int64_t off = row * a.row_stride + c;
    float g = __fmul_rn(uniq_grads[u * a.dim + c], h.grad_scale);
    float w = a.table[off];
    float s0 = a.state0 ? a.state0[off] : 0.f;
    float s1 = a.state1 ? a.state1[off] : 0.f;
    upd_one(a, h, g, w, s0, s1);
    a.table[off] = w;
    if (a.state0) a.state0[off] = s0;
    if (a.state1) a.state1[off] = s1;
  }
}

// TF AdamOptimizer on the rows that received no gradient this step: m *= b1, v *= b2,
// w -= lr_t*m/(sqrt(v)+eps) (the decay half of _apply_sparse_shared in TF's adam.py; behaviour stated at
// compat/adam_s.py:74-81).  Pure stream over the table: one thread per VEC floats of a row, rows whose
// moments are all zero are not written back (never-touched rows: the update is exactly 0).
struct SweepArgs {
  float* table;
  float* m;
  float* v;
  int64_t n_rows;
  int dim;
  int row_stride;
  const uint8_t* touched;
  er_opt_t opt;
  float lr_t;
  const float* hyper;
};

__device__ __forceinline__ void sweep_one(float& w, float& m, float& v, float b1, float b2, float eps, float lr_t) {
  m = __fmul_rn(m, b1);
  v = __fmul_rn(v, b2);
  w = __fsub_rn(w, __fdiv_rn(__fmul_rn(lr_t, m), __fadd_rn(__fsqrt_rn(v), eps)));
}

__global__ void __launch_bounds__(256) adam_sweep_vec_kernel(const __grid_constant__ SweepArgs a) {
  const Hyper h = load_hyper(a.opt, a.lr_t, a.hyper);
  const int d4 = a.dim >> 2;
  const int64_t total = a.n_rows * d4;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / d4;
    const int c = (int)(t - r * d4);
    if (a.touched && a.touched[r]) continue;
    const int64_t off = r * a.row_stride;
    float4* pm = reinterpret_cast<float4*>(a.m + off) + c;
    float4* pv = reinterpret_cast<float4*>(a.v + off) + c;
    float4 m = *pm, v = *pv;
    if (m.x == 0.f && m.y == 0.f && m.z == 0.f && m.w == 0.f && v.x == 0.f && v.y == 0.f && v.z == 0.f &&
        v.w == 0.f)
      continue;
    float4* pw = reinterpret_cast<float4*>(a.table + off) + c;
    float4 w = *pw;
    sweep_one(w.x, m.x, v.x, a.opt.beta1, a.opt.beta2, a.opt.eps, h.lr_t);
    sweep_one(w.y, m.y, v.y, a.opt.beta1, a.opt.beta2, a.opt.eps, h.lr_t);
    sweep_one(w.z, m.z, v.z, a.opt.beta1, a.opt.beta2, a.opt.eps, h.lr_t);
    sweep_one(w.w, m.w, v.w, a.opt.beta1, a.opt.beta2, a.opt.eps, h.lr_t);
    *pm = m;
    *pv = v;
    *pw = w;
  }
}

__global__ void __launch_bounds__(256) adam_sweep_kernel(const __grid_constant__ SweepArgs a) {
  const Hyper h = load_hyper(a.opt, a.lr_t, a.hyper);
  const int64_t total = a.n_rows * a.dim;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / a.dim;
    const int c = (int)(t - r * a.dim);
    if (a.touched && a.touched[r]) continue;
    const int64_t off = r * a.row_stride + c;
    float m = a.m[off], v = a.v[off];
    if (m == 0.f && v == 0.f) continue;
    float w = a.table[off];
    sweep_one(w, m, v, a.opt.beta1, a.opt.beta2, a.opt.eps, h.lr_t);
    a.m[off] = m;
    a.v[off] = v;
    a.table[off] = w;
  }
}

}  // namespace er

extern "C" int er_sparse_apply(float* table, float* state0, float* state1, int32_t dim,
                               int32_t row_stride, const int64_t* uniq_rows,
                               const float* uniq_grads, const int32_t* n_uniq, int64_t n_cap,
                               const er_opt_t* opt, er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(table && uniq_rows && uniq_grads && opt, "null argument");
  ER_REQUIRE(dim > 0 && row_stride >= dim, "bad dim / row_stride");
  const int k = opt->kind;
  ER_REQUIRE(k == ER_OPT_SGD || state0, "optimizer state0 missing");
  ER_REQUIRE((k != ER_OPT_LAZY_ADAM && k != ER_OPT_ADAM_ROWS) || state1, "adam needs state1 (v)");
  if (n_cap <= 0) return ER_OK;
  BwdArgs a = {};
  a.table = table;
  a.state0 = state0;
  a.state1 = state1;
  a.dim = dim;
  a.row_stride = row_stride;
  a.opt = *opt;
  a.lr_t = (k == ER_OPT_LAZY_ADAM || k == ER_OPT_ADAM_ROWS) ? adam_lr_t(*opt) : opt->lr;
  a.hyper = opt->hyper_dev;
  sparse_apply_kernel<<<grid_for(n_cap * dim, 256, 8), 256, 0, as_stream(stream)>>>(
      a, uniq_rows, uniq_grads, n_uniq, n_cap);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_adam_dense_sweep(float* table, float* m, float* v, int64_t n_rows, int32_t dim,
                                   int32_t row_stride, const uint8_t* touched,
                                   const er_opt_t* opt, er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(table && m && v && opt, "null argument");
  ER_REQUIRE(dim > 0 && row_stride >= dim && n_rows > 0, "bad shape");
  SweepArgs a;
  a.table = table;
  a.m = m;
  a.v = v;
  a.n_rows = n_rows;
  a.dim = dim;
  a.row_stride = row_stride;
  a.touched = touched;
  a.opt = *opt;
  a.opt.kind = ER_OPT_ADAM_ROWS;
  a.lr_t = adam_lr_t(*opt);
  a.hyper = opt->hyper_dev;
  const bool vec = dim % 4 == 0 && row_stride % 4 == 0 && reinterpret_cast<uintptr_t>(table) % 16 == 0 &&
                   reinterpret_cast<uintptr_t>(m) % 16 == 0 && reinterpret_cast<uintptr_t>(v) % 16 == 0;
  if (vec)
    adam_sweep_vec_kernel<<<grid_for(n_rows * (dim / 4), 256, 8), 256, 0, as_stream(stream)>>>(a);
  else
    adam_sweep_kernel<<<grid_for(n_rows * dim, 256, 8), 256, 0, as_stream(stream)>>>(a);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}
