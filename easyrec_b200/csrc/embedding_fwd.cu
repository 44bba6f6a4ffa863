// K2: multi-slot embedding gather + pool with the group concat fused into the
// store.  Replaces, per feature column of a group,
//   safe_embedding_lookup_sparse -> unique + gather + sparse_segment_{sum,mean,sqrtn}
//   -> reshape [B, D] -> concat axis 1
// (compat/embedding_ops.py:37-162; compat/feature_column/feature_column.py:202-244,
//  384-414) and the packed path's sparse_segment_sum + [N,B,D]->[B,N*D] transpose
// (feature_column.py:326-357).
//
// HBM-bound random row reads: one embedding row is dim*4 bytes (64 B at D=16 =
// two 32 B sectors).  A group of dim/4 lanes owns one segment and moves the row
// with one 16 B non-allocating load per lane; kUnroll independent segments per
// group are in flight before the first use so that each SM keeps >32 KB of row
// reads outstanding (Little's law at ~6.5 TB/s x ~600 ns needs ~26 KB/SM).
// Segment -> slot goes through the shared-memory SlotView (slots.cuh): one multiply-shift
// and one LDS.128 per segment.  Accumulation inside a segment is sequential in lookup
// order with separate multiply and add (no FMA contraction), i.e. the CPU reference's order.
#include "common.cuh"
#include "slots.cuh"

namespace er {

struct Bufs {
  float* p[ER_MAX_BUFS];
};

__device__ __forceinline__ float4 f4_zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ float4 f4_add(const float4& a, const float4& b) {
  return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z),
                     __fadd_rn(a.w, b.w));
}
__device__ __forceinline__ float4 f4_scale(const float4& a, float w) {
  return make_float4(__fmul_rn(a.x, w), __fmul_rn(a.y, w), __fmul_rn(a.z, w), __fmul_rn(a.w, w));
}
__device__ __forceinline__ float4 f4_div(const float4& a, float d) {
  return make_float4(__fdiv_rn(a.x, d), __fdiv_rn(a.y, d), __fdiv_rn(a.z, d), __fdiv_rn(a.w, d));
}

// ---- fast path: every segment holds exactly one lookup (row_ptr == NULL) ----
template <int LANES, int UNROLL>
__global__ void __launch_bounds__(256)
    fwd_single_kernel(const float* __restrict__ table, int row_stride,
                      const int64_t* __restrict__ rows, const float* __restrict__ weights,
                      int64_t n_seg, const er_slot_t* __restrict__ slots, int n_slots,
                      const __grid_constant__ Bufs bufs, float* __restrict__ seg_scale) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  const SlotView sv = load_slots(s_raw, slots, n_slots);
  const int lane = threadIdx.x % LANES;
  const int64_t n_groups = (int64_t)gridDim.x * (blockDim.x / LANES);
  const int64_t g = (int64_t)blockIdx.x * (blockDim.x / LANES) + threadIdx.x / LANES;
  for (int64_t base = 0; base < n_seg; base += n_groups * UNROLL) {
    int64_t r[UNROLL];
    float w[UNROLL];
    float4 v[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const int64_t s = base + (int64_t)u * n_groups + g;
      r[u] = (s < n_seg) ? rows[s] : -1;
      w[u] = (weights && s < n_seg) ? weights[s] : 1.0f;
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      v[u] = f4_zero();
      if (r[u] >= 0)
        v[u] = ld_row_f4(reinterpret_cast<const float4*>(table + r[u] * (int64_t)row_stride) + lane);
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const int64_t s = base + (int64_t)u * n_groups + g;
      if (s >= n_seg) continue;
      const SlotLite sl = slot_lite(sv, slot_of(sv, (int32_t)s));
      const int comb = slot_comb(sl);
      float4 o = f4_zero();
      float scale = comb == ER_COMBINER_SUM ? 1.f : 0.f;   // sum: 1 for every segment, as the CSR and scalar paths
      const bool keep = r[u] >= 0 && (comb == ER_COMBINER_SUM || w[u] > 0.f);
      if (keep) {
        o = weights ? f4_scale(v[u], w[u]) : v[u];
        if (comb == ER_COMBINER_MEAN) {
          o = f4_div(o, w[u]);
          scale = __fdiv_rn(1.f, w[u]);
        } else if (comb == ER_COMBINER_SQRTN) {
          const float d = sqrtf(__fmul_rn(w[u], w[u]));   // 0 when w*w underflows: zeros, as the CSR path
          o = d != 0.f ? f4_div(o, d) : f4_zero();
          scale = d != 0.f ? __fdiv_rn(1.f, d) : 0.f;
        }
      }
      float* dst = bufs.p[sl.misc & 0xff] + (int64_t)((int32_t)s - sl.seg_begin) * sl.out_stride + sl.out_col;
      reinterpret_cast<float4*>(dst)[lane] = o;
      if (seg_scale && lane == 0) seg_scale[s] = scale;
    }
  }
}

// ---- general CSR path: variable-length, weighted segments ----
template <int LANES>
__global__ void __launch_bounds__(256)
    fwd_csr_kernel(const float* __restrict__ table, int row_stride,
                   const int64_t* __restrict__ rows, const float* __restrict__ weights,
                   const int32_t* __restrict__ row_ptr, int64_t n_seg, int64_t cap,
                   const er_slot_t* __restrict__ slots, int n_slots,
                   const __grid_constant__ Bufs bufs, float* __restrict__ seg_scale) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  const SlotView sv = load_slots(s_raw, slots, n_slots);
  const int lane = threadIdx.x % LANES;
  const int64_t n_groups = (int64_t)gridDim.x * (blockDim.x / LANES);
  const int64_t g = (int64_t)blockIdx.x * (blockDim.x / LANES) + threadIdx.x / LANES;
  constexpr int U = 4;
  for (int64_t s = g; s < n_seg; s += n_groups) {
    const SlotLite sl = slot_lite(sv, slot_of(sv, (int32_t)s));
    const int comb = slot_comb(sl);
    int64_t b = row_ptr[s], e = row_ptr[s + 1];
    if (e > cap) e = cap;
    float4 acc = f4_zero();
    float wsum = 0.f, w2sum = 0.f;
    const bool is_sum = comb == ER_COMBINER_SUM;
    for (int64_t j = b; j < e; j += U) {
      int64_t r[U];
      float w[U];
      float4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        r[u] = (j + u < e) ? rows[j + u] : -1;
        w[u] = (weights && j + u < e) ? weights[j + u] : 1.0f;
        if (!is_sum && !(w[u] > 0.f)) r[u] = -1;  // _prune_invalid_weights
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        v[u] = f4_zero();
        if (r[u] >= 0)
          v[u] = ld_row_f4(reinterpret_cast<const float4*>(table + r[u] * (int64_t)row_stride) + lane);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (r[u] < 0) continue;
        acc = f4_add(acc, weights ? f4_scale(v[u], w[u]) : v[u]);
        wsum = __fadd_rn(wsum, w[u]);
        w2sum = __fadd_rn(w2sum, __fmul_rn(w[u], w[u]));
      }
    }
    float scale = 1.f;
    if (comb == ER_COMBINER_MEAN) {
      if (wsum != 0.f) {
        acc = f4_div(acc, wsum);
        scale = __fdiv_rn(1.f, wsum);
      } else {
        acc = f4_zero();
        scale = 0.f;
      }
    } else if (comb == ER_COMBINER_SQRTN) {
      const float d = sqrtf(w2sum);
      if (d != 0.f) {
        acc = f4_div(acc, d);
        scale = __fdiv_rn(1.f, d);
      } else {
        acc = f4_zero();
        scale = 0.f;
      }
    }
    float* dst = bufs.p[sl.misc & 0xff] + (int64_t)((int32_t)s - sl.seg_begin) * sl.out_stride + sl.out_col;
    reinterpret_cast<float4*>(dst)[lane] = acc;
    if (seg_scale && lane == 0) seg_scale[s] = scale;
  }
}

// ---- scalar path: any dim (wide dim=1 tables, odd dims); one thread per (segment, column) ----
__global__ void __launch_bounds__(256)
    fwd_scalar_kernel(const float* __restrict__ table, int dim, int row_stride,
                      const int64_t* __restrict__ rows, const float* __restrict__ weights,
                      const int32_t* __restrict__ row_ptr, int64_t n_seg, int64_t cap,
                      const er_slot_t* __restrict__ slots, int n_slots,
                      const __grid_constant__ Bufs bufs, float* __restrict__ seg_scale) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  const SlotView sv = load_slots(s_raw, slots, n_slots);
  const FastDiv ddiv = make_fastdiv((uint32_t)dim);
  const int64_t total = n_seg * dim;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t s = (total < (1LL << 32)) ? (int64_t)fastdiv((uint32_t)t, ddiv) : t / dim;
    const int c = (int)(t - s * dim);
    const SlotLite sl = slot_lite(sv, slot_of(sv, (int32_t)s));
    const int comb = slot_comb(sl);
    int64_t b = row_ptr ? row_ptr[s] : s, e = row_ptr ? row_ptr[s + 1] : s + 1;
    if (e > cap) e = cap;
    const bool is_sum = comb == ER_COMBINER_SUM;
    float acc = 0.f, wsum = 0.f, w2sum = 0.f;
    for (int64_t j = b; j < e; ++j) {
      const int64_t r = rows[j];
      const float w = weights ? weights[j] : 1.0f;
      if (r < 0 || (!is_sum && !(w > 0.f))) continue;
      const float v = __ldg(table + r * (int64_t)row_stride + c);
      acc = __fadd_rn(acc, weights ? __fmul_rn(v, w) : v);
      wsum = __fadd_rn(wsum, w);
      w2sum = __fadd_rn(w2sum, __fmul_rn(w, w));
    }
    float scale = 1.f;
    if (comb == ER_COMBINER_MEAN) {
      scale = wsum != 0.f ? __fdiv_rn(1.f, wsum) : 0.f;
      acc = wsum != 0.f ? __fdiv_rn(acc, wsum) : 0.f;
    } else if (comb == ER_COMBINER_SQRTN) {
      const float d = sqrtf(w2sum);
      scale = d != 0.f ? __fdiv_rn(1.f, d) : 0.f;
      acc = d != 0.f ? __fdiv_rn(acc, d) : 0.f;
    }
    bufs.p[sl.misc & 0xff][(int64_t)((int32_t)s - sl.seg_begin) * sl.out_stride + sl.out_col + c] = acc;
    if (seg_scale && c == 0) seg_scale[s] = scale;
  }
}

template <int LANES>
static void launch_vec(const float* table, int row_stride, const int64_t* rows,
                       const float* weights, const int32_t* row_ptr, int64_t n_seg, int64_t cap,
                       const er_slot_t* slots, int n_slots, const Bufs& bufs, float* seg_scale,
                       cudaStream_t st) {
  const size_t smem = slot_smem_bytes(n_slots);
  const int groups_per_cta = 256 / LANES;
  if (!row_ptr) {
    constexpr int UNROLL = 4;
    int grid = grid_for(ceil_div(n_seg, UNROLL), groups_per_cta, 8);
    fwd_single_kernel<LANES, UNROLL><<<grid, 256, smem, st>>>(table, row_stride, rows, weights,
                                                              n_seg, slots, n_slots, bufs, seg_scale);
  } else {
    int grid = grid_for(n_seg, groups_per_cta, 8);
    fwd_csr_kernel<LANES><<<grid, 256, smem, st>>>(table, row_stride, rows, weights, row_ptr, n_seg,
                                                   cap, slots, n_slots, bufs, seg_scale);
  }
}

}  // namespace er

extern "C" int er_embedding_fwd(const float* table, int64_t n_rows, int32_t dim,
                                int32_t row_stride, const int64_t* rows, const float* weights,
                                const int32_t* row_ptr, int64_t n_seg, int64_t n_lookups_cap,
                                const er_slot_t* slots, int32_t n_slots, float* const* out_bufs,
                                int32_t n_bufs, float* seg_scale, er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(table && rows && slots && out_bufs, "null argument");
  ER_REQUIRE(dim > 0 && row_stride >= dim, "bad dim / row_stride");
  ER_REQUIRE(n_rows > 0, "n_rows must be positive");
  ER_REQUIRE(n_slots > 0 && n_slots <= 2048, "n_slots must be in [1, 2048]");
  ER_REQUIRE(n_bufs > 0 && n_bufs <= ER_MAX_BUFS, "n_bufs must be in [1, ER_MAX_BUFS]");
  ER_REQUIRE(n_seg >= 0 && n_seg < (1LL << 31), "n_seg out of range");
  ER_REQUIRE(row_ptr || n_lookups_cap == n_seg,
             "row_ptr == NULL requires n_lookups_cap == n_seg (single-valued slots)");
  if (n_seg == 0) return ER_OK;
  Bufs bufs;
  bool aligned = (reinterpret_cast<uintptr_t>(table) % 16 == 0) && (row_stride % 4 == 0);
  for (int i = 0; i < ER_MAX_BUFS; ++i) {
    bufs.p[i] = i < n_bufs ? out_bufs[i] : nullptr;
    if (i < n_bufs) {
      ER_REQUIRE(out_bufs[i] != nullptr, "null output buffer");
      aligned = aligned && (reinterpret_cast<uintptr_t>(out_bufs[i]) % 16 == 0);
    }
  }
  cudaStream_t st = as_stream(stream);
  const bool vec_dim = (dim == 4 || dim == 8 || dim == 16 || dim == 32 || dim == 64 || dim == 128);
  // the host plan guarantees out_stride % 4 == 0 and out_col % 4 == 0 for vector dims
  // (K.make_slots refuses other plans); the scalar path has no alignment requirement.
  if (vec_dim && aligned) {
    switch (dim / 4) {
      case 1: launch_vec<1>(table, row_stride, rows, weights, row_ptr, n_seg, n_lookups_cap, slots, n_slots, bufs, seg_scale, st); break;
      case 2: launch_vec<2>(table, row_stride, rows, weights, row_ptr, n_seg, n_lookups_cap, slots, n_slots, bufs, seg_scale, st); break;
      case 4: launch_vec<4>(table, row_stride, rows, weights, row_ptr, n_seg, n_lookups_cap, slots, n_slots, bufs, seg_scale, st); break;
      case 8: launch_vec<8>(table, row_stride, rows, weights, row_ptr, n_seg, n_lookups_cap, slots, n_slots, bufs, seg_scale, st); break;
      case 16: launch_vec<16>(table, row_stride, rows, weights, row_ptr, n_seg, n_lookups_cap, slots, n_slots, bufs, seg_scale, st); break;
      default: launch_vec<32>(table, row_stride, rows, weights, row_ptr, n_seg, n_lookups_cap, slots, n_slots, bufs, seg_scale, st); break;
    }
  } else {
    int grid = grid_for(n_seg * (int64_t)dim, 256, 8);
    fwd_scalar_kernel<<<grid, 256, slot_smem_bytes(n_slots), st>>>(
        table, dim, row_stride, rows, weights, row_ptr, n_seg, n_lookups_cap, slots, n_slots, bufs,
        seg_scale);
  }
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}
