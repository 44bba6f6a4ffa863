// K6 epilogues: the non-GEMM part of EasyRec's DNN layer (layers/dnn.py:56-79)
//     z = x W + b ;  h = batch_norm(z) ;  y = relu(h)
// fused into two launches forward and two backward, fp32, deterministic.
//   tf.layers.batch_normalization defaults: momentum 0.99, epsilon 1e-3, batch statistics in
//   training with the BIASED variance for both the normalisation and the moving average.
// The GEMMs are er_gemm (gemm.cu, wgmma) / er_gemm_small (small_gemm.cu).
//
// Decomposition: 32-column tiles x R row chunks (grid ~ 2 waves of the 132 SMs).  Pass 1 writes
// per-chunk partial statistics (Welford count/mean/M2, merged with Chan's formula in a fixed order
// -- no atomics, no E[x^2]-E[x]^2 cancellation); pass 2 re-derives the column statistics from the
// R partials (R*32 L2 reads per CTA) and streams the tile.  Traffic: fwd 2 reads + 1 write of
// [B,U]; bwd 3 reads (z, y, gy) twice + 1 write.  er_bn_relu_bwd recomputes the relu mask from z (bn_pre_act) instead
// of reading y: 2 reads (z, gy) twice + 1 write.
#include <algorithm>

#include "common.cuh"
#include "elementwise.cuh"

namespace er {

constexpr int kColTile = 32;
constexpr int kRowLanes = 8;  // 256 threads = 32 columns x 8 row lanes

struct Welford {
  float n, mean, m2;
};
__device__ __forceinline__ void wf_merge(Welford& a, const Welford& b) {
  if (b.n == 0.f) return;
  const float n = a.n + b.n;
  const float d = b.mean - a.mean;
  a.mean += d * (b.n / n);
  a.m2 += b.m2 + d * d * (a.n * b.n / n);
  a.n = n;
}

struct DenseShape {
  int64_t batch;
  int units;
  int rows_per_chunk;
  int n_chunks;
};

inline DenseShape dense_shape(int64_t batch, int units) {
  DenseShape s;
  s.batch = batch;
  s.units = units;
  const int col_tiles = (units + kColTile - 1) / kColTile;
  int r = (2 * kSmCount + col_tiles - 1) / col_tiles;
  if (r < 1) r = 1;
  int64_t rpc = ceil_div(batch, (int64_t)r);
  rpc = ceil_div(rpc, (int64_t)kRowLanes) * kRowLanes;
  if (rpc < kRowLanes) rpc = kRowLanes;
  s.rows_per_chunk = (int)rpc;
  s.n_chunks = (int)ceil_div(batch, rpc);
  return s;
}

// ---- forward pass 1: partial statistics of z + b ----
__global__ void __launch_bounds__(256)
    bn_stats_kernel(const float* __restrict__ z, const float* __restrict__ bias, DenseShape s,
                    float* __restrict__ part /* [n_chunks][units][3] */) {
  __shared__ Welford s_w[kRowLanes][kColTile];
  const int c = blockIdx.x * kColTile + (threadIdx.x & 31);
  const int rl = threadIdx.x >> 5;
  const int64_t r0 = (int64_t)blockIdx.y * s.rows_per_chunk;
  const int64_t r1 = min(s.batch, r0 + s.rows_per_chunk);
  Welford w = {0.f, 0.f, 0.f};
  if (c < s.units && r0 + rl < r1) {
    // shifted sums (shift = first value of the lane) -> (n, mean, M2): no per-element division,
    // and no E[x^2]-E[x]^2 cancellation because the shift sits next to the mean
    const float b = bias ? bias[c] : 0.f;
    const float shift = z[(r0 + rl) * s.units + c] + b;
    float n = 0.f, sm = 0.f, sq = 0.f;
    for (int64_t r = r0 + rl; r < r1; r += kRowLanes) {
      const float d = (z[r * s.units + c] + b) - shift;
      n += 1.f;
      sm += d;
      sq += d * d;
    }
    w.n = n;
    w.mean = shift + sm / n;
    w.m2 = sq - sm * sm / n;
  }
  s_w[rl][threadIdx.x & 31] = w;
  __syncthreads();
  if (rl == 0 && c < s.units) {
    Welford t = s_w[0][threadIdx.x];
    for (int k = 1; k < kRowLanes; ++k) wf_merge(t, s_w[k][threadIdx.x]);
    float* p = part + ((int64_t)blockIdx.y * s.units + c) * 3;
    p[0] = t.n;
    p[1] = t.mean;
    p[2] = t.m2;
  }
}

// ---- forward pass 2: merge partials, normalise, activation ----
__global__ void __launch_bounds__(256)
    bn_apply_kernel(const float* __restrict__ z, const float* __restrict__ bias,
                    const float* __restrict__ gamma, const float* __restrict__ beta,
                    float* __restrict__ moving_mean, float* __restrict__ moving_var, DenseShape s,
                    float eps, float momentum, int training, int relu, const float* __restrict__ part,
                    float* __restrict__ y, float* __restrict__ save_mean, float* __restrict__ save_rstd) {
  __shared__ float s_mean[kColTile], s_rstd[kColTile];
  __shared__ Welford s_m[kRowLanes][kColTile];
  const int c = blockIdx.x * kColTile + (threadIdx.x & 31);
  const int rl = threadIdx.x >> 5;
  if (training) {  // the 8 row lanes merge the chunk partials in parallel, then lane 0 merges the 8
    Welford t = {0.f, 0.f, 0.f};
    if (c < s.units) {
      for (int k = rl; k < s.n_chunks; k += kRowLanes) {
        const float* p = part + ((int64_t)k * s.units + c) * 3;
        Welford q = {p[0], p[1], p[2]};
        wf_merge(t, q);
      }
    }
    s_m[rl][threadIdx.x & 31] = t;
    __syncthreads();
  }
  if (rl == 0 && c < s.units) {
    float mean, var;
    if (training) {
      Welford t = s_m[0][threadIdx.x];
      for (int k = 1; k < kRowLanes; ++k) wf_merge(t, s_m[k][threadIdx.x]);
      mean = t.mean;
      var = t.m2 / t.n;  // biased
      if (blockIdx.y == 0) {
        moving_mean[c] = moving_mean[c] * momentum + mean * (1.f - momentum);
        moving_var[c] = moving_var[c] * momentum + var * (1.f - momentum);
      }
    } else {
      mean = moving_mean[c];
      var = moving_var[c];
    }
    const float rstd = 1.0f / sqrtf(var + eps);
    s_mean[threadIdx.x] = mean;
    s_rstd[threadIdx.x] = rstd;
    if (blockIdx.y == 0 && save_mean) {
      save_mean[c] = mean;
      save_rstd[c] = rstd;
    }
  }
  __syncthreads();
  if (c >= s.units) return;
  const float b = bias ? bias[c] : 0.f;
  const float mean = s_mean[threadIdx.x & 31], rstd = s_rstd[threadIdx.x & 31];
  const float ga = gamma[c], be = beta[c];
  const int64_t r0 = (int64_t)blockIdx.y * s.rows_per_chunk;
  const int64_t r1 = min(s.batch, r0 + s.rows_per_chunk);
  for (int64_t r = r0 + rl; r < r1; r += kRowLanes) {
    const float h = bn_pre_act(z[r * s.units + c], b, mean, rstd, ga, be);
    y[r * s.units + c] = relu ? fmaxf(h, 0.f) : h;
  }
}

// y = act(bn(z + b)) with known column statistics: one streaming pass, 16 B per thread access
__global__ void __launch_bounds__(256)
    bn_act_apply_vec_kernel(const float4* __restrict__ z, const float* __restrict__ bias,
                            const float* __restrict__ gamma, const float* __restrict__ beta,
                            const float* __restrict__ mean, const float* __restrict__ rstd, int64_t total4,
                            int units, int relu, float4* __restrict__ y) {
  er_pdl_wait();
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total4;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)((t * 4) % units);
    const float4 v = z[t];
    const float4 mu = *reinterpret_cast<const float4*>(mean + c);
    const float4 rs = *reinterpret_cast<const float4*>(rstd + c);
    const float4 ga = *reinterpret_cast<const float4*>(gamma + c);
    const float4 be = *reinterpret_cast<const float4*>(beta + c);
    float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
    if (bias) b = *reinterpret_cast<const float4*>(bias + c);
    float4 h;
    h.x = bn_pre_act(v.x, b.x, mu.x, rs.x, ga.x, be.x);
    h.y = bn_pre_act(v.y, b.y, mu.y, rs.y, ga.y, be.y);
    h.z = bn_pre_act(v.z, b.z, mu.z, rs.z, ga.z, be.z);
    h.w = bn_pre_act(v.w, b.w, mu.w, rs.w, ga.w, be.w);
    if (relu) {
      h.x = fmaxf(h.x, 0.f); h.y = fmaxf(h.y, 0.f); h.z = fmaxf(h.z, 0.f); h.w = fmaxf(h.w, 0.f);
    }
    y[t] = h;
  }
}
__global__ void __launch_bounds__(256)
    bn_act_apply_kernel(const float* __restrict__ z, const float* __restrict__ bias,
                        const float* __restrict__ gamma, const float* __restrict__ beta,
                        const float* __restrict__ mean, const float* __restrict__ rstd, int64_t total,
                        int units, int relu, float* __restrict__ y) {
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(t % units);
    const float h = bn_pre_act(z[t], bias ? bias[c] : 0.f, mean[c], rstd[c], gamma[c], beta[c]);
    y[t] = relu ? fmaxf(h, 0.f) : h;
  }
}

// no batch norm: y = act(z + b)
__global__ void __launch_bounds__(256)
    bias_act_kernel(const float* __restrict__ z, const float* __restrict__ bias, int64_t total, int units,
                    int relu, float* __restrict__ y) {
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const float h = z[t] + (bias ? bias[t % units] : 0.f);
    y[t] = relu ? fmaxf(h, 0.f) : h;
  }
}

// ---- backward pass 1: partial column sums of g and g*xhat (BN) or of g (no BN) ----
__global__ void __launch_bounds__(256)
    bn_bwd_stats_kernel(const float* __restrict__ z, const float* __restrict__ bias,
                        const float* __restrict__ y, const float* __restrict__ gy,
                        const float* __restrict__ save_mean, const float* __restrict__ save_rstd,
                        DenseShape s, int relu, int use_bn, float* __restrict__ part /* [n_chunks][units][2] */) {
  __shared__ float s_a[kRowLanes][kColTile], s_b[kRowLanes][kColTile];
  const int c = blockIdx.x * kColTile + (threadIdx.x & 31);
  const int rl = threadIdx.x >> 5;
  const int64_t r0 = (int64_t)blockIdx.y * s.rows_per_chunk;
  const int64_t r1 = min(s.batch, r0 + s.rows_per_chunk);
  float sg = 0.f, sgx = 0.f;
  if (c < s.units) {
    const float b = bias ? bias[c] : 0.f;
    const float mean = use_bn ? save_mean[c] : 0.f, rstd = use_bn ? save_rstd[c] : 0.f;
    for (int64_t r = r0 + rl; r < r1; r += kRowLanes) {
      const int64_t i = r * s.units + c;
      float g = gy[i];
      if (relu && !(y[i] > 0.f)) g = 0.f;
      sg += g;
      if (use_bn) sgx += g * (((z[i] + b) - mean) * rstd);
    }
  }
  s_a[rl][threadIdx.x & 31] = sg;
  s_b[rl][threadIdx.x & 31] = sgx;
  __syncthreads();
  if (rl == 0 && c < s.units) {
    float a = s_a[0][threadIdx.x], bb = s_b[0][threadIdx.x];
    for (int k = 1; k < kRowLanes; ++k) {
      a += s_a[k][threadIdx.x];
      bb += s_b[k][threadIdx.x];
    }
    float* p = part + ((int64_t)blockIdx.y * s.units + c) * 2;
    p[0] = a;
    p[1] = bb;
  }
}

// ---- backward pass 2: gz = gamma*rstd*(g - dbeta/B - xhat*dgamma/B)  (BN)   |   gz = g ----
__global__ void __launch_bounds__(256)
    bn_bwd_apply_kernel(const float* __restrict__ z, const float* __restrict__ bias,
                        const float* __restrict__ gamma, const float* __restrict__ y,
                        const float* __restrict__ gy, const float* __restrict__ save_mean,
                        const float* __restrict__ save_rstd, DenseShape s, int relu, int use_bn,
                        const float* __restrict__ part, float* __restrict__ gz,
                        float* __restrict__ gbias, float* __restrict__ ggamma, float* __restrict__ gbeta) {
  __shared__ float s_dg[kColTile], s_db[kColTile];
  __shared__ float s_pa[kRowLanes][kColTile], s_pb[kRowLanes][kColTile];
  const int c = blockIdx.x * kColTile + (threadIdx.x & 31);
  const int rl = threadIdx.x >> 5;
  {  // the 8 row lanes add the chunk partials in parallel (fixed order), lane 0 adds the 8
    float a = 0.f, b = 0.f;
    if (c < s.units) {
      for (int k = rl; k < s.n_chunks; k += kRowLanes) {
        const float* p = part + ((int64_t)k * s.units + c) * 2;
        a += p[0];
        b += p[1];
      }
    }
    s_pa[rl][threadIdx.x & 31] = a;
    s_pb[rl][threadIdx.x & 31] = b;
    __syncthreads();
  }
  if (rl == 0 && c < s.units) {
    float a = 0.f, b = 0.f;
    for (int k = 0; k < kRowLanes; ++k) {
      a += s_pa[k][threadIdx.x];
      b += s_pb[k][threadIdx.x];
    }
    s_db[threadIdx.x] = a;  // sum g
    s_dg[threadIdx.x] = b;  // sum g*xhat
    if (blockIdx.y == 0) {
      if (use_bn) {
        if (ggamma) ggamma[c] = b;
        if (gbeta) gbeta[c] = a;
        // d/dbias of a batch-normalised pre-activation is identically zero (BN removes the mean);
        // TF evaluates it as rounding noise ~1e-9.
        if (gbias) gbias[c] = 0.f;
      } else if (gbias) {
        gbias[c] = a;
      }
    }
  }
  __syncthreads();
  if (c >= s.units) return;
  const float bsum = s_db[threadIdx.x & 31], gsum = s_dg[threadIdx.x & 31];
  const float bv = bias ? bias[c] : 0.f;
  const float mean = use_bn ? save_mean[c] : 0.f, rstd = use_bn ? save_rstd[c] : 0.f;
  const float ga = use_bn ? gamma[c] : 1.f;
  const float inv_b = 1.0f / (float)s.batch;
  const int64_t r0 = (int64_t)blockIdx.y * s.rows_per_chunk;
  const int64_t r1 = min(s.batch, r0 + s.rows_per_chunk);
  for (int64_t r = r0 + rl; r < r1; r += kRowLanes) {
    const int64_t i = r * s.units + c;
    float g = gy[i];
    if (relu && !(y[i] > 0.f)) g = 0.f;
    if (use_bn) {
      const float xhat = ((z[i] + bv) - mean) * rstd;
      g = ga * rstd * (g - bsum * inv_b - xhat * gsum * inv_b);
    }
    gz[i] = g;
  }
}

// ---- vector backward (units % 4 == 0): the same two passes with 16-byte accesses --------------------
// CTA = 128 columns (32 float4 lanes) x 8 row lanes over one row chunk; one wave of CTAs.  Pass 1 writes one
// (sum g, sum g*xhat) partial per (chunk, column); pass 2's CTAs each re-add the chunk partials of their
// 128 columns (8 row lanes in parallel, fixed order: deterministic, no tickets, no atomics) and stream.
constexpr int kVecCols = 128;

struct VecShape {
  int64_t batch;
  int units;
  int rows_per_chunk;
  int n_chunks;
};
inline VecShape vec_shape(int64_t batch, int units) {
  VecShape s;
  s.batch = batch;
  s.units = units;
  const int col_tiles = (units + kVecCols - 1) / kVecCols;
  const int r = std::max(1, (kSmCount + col_tiles - 1) / col_tiles);
  int64_t rpc = ceil_div(batch, (int64_t)r);
  rpc = std::max<int64_t>(ceil_div(rpc, (int64_t)kRowLanes) * kRowLanes, 2 * kRowLanes);
  s.rows_per_chunk = (int)rpc;
  s.n_chunks = (int)ceil_div(batch, rpc);
  return s;
}

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void relu_mask4(float4& g, const float4& yy) {
  if (!(yy.x > 0.f)) g.x = 0.f;
  if (!(yy.y > 0.f)) g.y = 0.f;
  if (!(yy.z > 0.f)) g.z = 0.f;
  if (!(yy.w > 0.f)) g.w = 0.f;
}
// the same mask from z: y > 0 exactly when the batch-normalised value is (bn_pre_act is the forward's expression)
__device__ __forceinline__ void relu_mask4_z(float4& g, const float4& zz, const float4& b, const float4& mu,
                                             const float4& rs, const float4& ga, const float4& be) {
  if (!(bn_pre_act(zz.x, b.x, mu.x, rs.x, ga.x, be.x) > 0.f)) g.x = 0.f;
  if (!(bn_pre_act(zz.y, b.y, mu.y, rs.y, ga.y, be.y) > 0.f)) g.y = 0.f;
  if (!(bn_pre_act(zz.z, b.z, mu.z, rs.z, ga.z, be.z) > 0.f)) g.z = 0.f;
  if (!(bn_pre_act(zz.w, b.w, mu.w, rs.w, ga.w, be.w) > 0.f)) g.w = 0.f;
}

// kZMask: batch norm + relu with the mask recomputed from z (gamma, beta given, y not read); else the mask comes from y
template <bool kZMask>
__global__ void __launch_bounds__(256)
    bn_bwd_stats_vec_kernel(const float* __restrict__ z, const float* __restrict__ bias,
                            const float* __restrict__ gamma, const float* __restrict__ beta,
                            const float* __restrict__ y, const float* __restrict__ gy,
                            const float* __restrict__ save_mean, const float* __restrict__ save_rstd,
                            VecShape s, int relu, int use_bn, float* __restrict__ part /* [n_chunks][units][2] */) {
  er_pdl_wait();
  __shared__ float4 s_a[kRowLanes][32], s_b[kRowLanes][32];
  const int cl = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int c = blockIdx.x * kVecCols + 4 * cl;
  const int64_t r0 = (int64_t)blockIdx.y * s.rows_per_chunk;
  const int64_t r1 = min(s.batch, r0 + s.rows_per_chunk);
  float4 sg = make_float4(0.f, 0.f, 0.f, 0.f), sx = sg;
  if (c < s.units) {
    float4 b = make_float4(0.f, 0.f, 0.f, 0.f), mu = b, rs = b, ga = b, be = b;
    if (bias) b = ld4(bias + c);
    if (use_bn) {
      mu = ld4(save_mean + c);
      rs = ld4(save_rstd + c);
    }
    if (kZMask) {
      ga = ld4(gamma + c);
      be = ld4(beta + c);
    }
#pragma unroll 4
    for (int64_t r = r0 + rl; r < r1; r += kRowLanes) {
      const int64_t i = r * s.units + c;
      float4 g = ld4(gy + i);
      if (kZMask) {
        if (relu) relu_mask4_z(g, ld4(z + i), b, mu, rs, ga, be);
      } else if (relu) {
        relu_mask4(g, ld4(y + i));
      }
      sg.x += g.x; sg.y += g.y; sg.z += g.z; sg.w += g.w;
      if (use_bn) {
        const float4 zz = ld4(z + i);
        sx.x += g.x * (((zz.x + b.x) - mu.x) * rs.x);
        sx.y += g.y * (((zz.y + b.y) - mu.y) * rs.y);
        sx.z += g.z * (((zz.z + b.z) - mu.z) * rs.z);
        sx.w += g.w * (((zz.w + b.w) - mu.w) * rs.w);
      }
    }
  }
  s_a[rl][cl] = sg;
  s_b[rl][cl] = sx;
  __syncthreads();
  if (rl == 0 && c < s.units) {
    float4 a = s_a[0][cl], bb = s_b[0][cl];
    for (int k = 1; k < kRowLanes; ++k) {
      const float4 p = s_a[k][cl], q = s_b[k][cl];
      a.x += p.x; a.y += p.y; a.z += p.z; a.w += p.w;
      bb.x += q.x; bb.y += q.y; bb.z += q.z; bb.w += q.w;
    }
    float4* p = reinterpret_cast<float4*>(part + ((int64_t)blockIdx.y * s.units + c) * 2);
    p[0] = a;    // sum g   of columns c..c+3
    p[1] = bb;   // sum g*xhat
  }
}

template <bool kZMask>
__global__ void __launch_bounds__(256)
    bn_bwd_apply_vec_kernel(const float* __restrict__ z, const float* __restrict__ bias,
                            const float* __restrict__ gamma, const float* __restrict__ beta,
                            const float* __restrict__ y, const float* __restrict__ gy,
                            const float* __restrict__ save_mean, const float* __restrict__ save_rstd, VecShape s,
                            int relu, int use_bn, const float* __restrict__ part, float* __restrict__ gz,
                            float* __restrict__ gbias, float* __restrict__ ggamma, float* __restrict__ gbeta) {
  er_pdl_wait();
  __shared__ float4 s_a[kRowLanes][32], s_b[kRowLanes][32];
  const int cl = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int c = blockIdx.x * kVecCols + 4 * cl;
  {  // the 8 row lanes add the chunk partials in parallel (chunks rl, rl+8, ...), lane 0 adds the 8
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    if (c < s.units) {
#pragma unroll 4
      for (int k = rl; k < s.n_chunks; k += kRowLanes) {
        const float4* p = reinterpret_cast<const float4*>(part + ((int64_t)k * s.units + c) * 2);
        const float4 pa = p[0], pb = p[1];
        a.x += pa.x; a.y += pa.y; a.z += pa.z; a.w += pa.w;
        b.x += pb.x; b.y += pb.y; b.z += pb.z; b.w += pb.w;
      }
    }
    s_a[rl][cl] = a;
    s_b[rl][cl] = b;
    __syncthreads();
  }
  float4 sg = s_a[0][cl], sx = s_b[0][cl];
  for (int k = 1; k < kRowLanes; ++k) {
    const float4 p = s_a[k][cl], q = s_b[k][cl];
    sg.x += p.x; sg.y += p.y; sg.z += p.z; sg.w += p.w;
    sx.x += q.x; sx.y += q.y; sx.z += q.z; sx.w += q.w;
  }
  if (c >= s.units) return;
  if (blockIdx.y == 0 && rl == 0) {
    if (use_bn) {
      if (ggamma) *reinterpret_cast<float4*>(ggamma + c) = sx;
      if (gbeta) *reinterpret_cast<float4*>(gbeta + c) = sg;
      if (gbias) *reinterpret_cast<float4*>(gbias + c) = make_float4(0.f, 0.f, 0.f, 0.f);   // see scalar kernel
    } else if (gbias) {
      *reinterpret_cast<float4*>(gbias + c) = sg;
    }
  }
  float4 b = make_float4(0.f, 0.f, 0.f, 0.f), mu = b, rs = b, be = b, ga = make_float4(1.f, 1.f, 1.f, 1.f);
  if (bias) b = ld4(bias + c);
  if (use_bn) {
    mu = ld4(save_mean + c);
    rs = ld4(save_rstd + c);
    ga = ld4(gamma + c);
  }
  if (kZMask) be = ld4(beta + c);
  const float inv_b = 1.0f / (float)s.batch;
  const int64_t r0 = (int64_t)blockIdx.y * s.rows_per_chunk;
  const int64_t r1 = min(s.batch, r0 + s.rows_per_chunk);
#pragma unroll 4
  for (int64_t r = r0 + rl; r < r1; r += kRowLanes) {
    const int64_t i = r * s.units + c;
    float4 g = ld4(gy + i);
    if (kZMask) {
      if (relu) relu_mask4_z(g, ld4(z + i), b, mu, rs, ga, be);
    } else if (relu) {
      relu_mask4(g, ld4(y + i));
    }
    if (use_bn) {
      const float4 zz = ld4(z + i);
      g.x = ga.x * rs.x * (g.x - sg.x * inv_b - (((zz.x + b.x) - mu.x) * rs.x) * sx.x * inv_b);
      g.y = ga.y * rs.y * (g.y - sg.y * inv_b - (((zz.y + b.y) - mu.y) * rs.y) * sx.y * inv_b);
      g.z = ga.z * rs.z * (g.z - sg.z * inv_b - (((zz.z + b.z) - mu.z) * rs.z) * sx.z * inv_b);
      g.w = ga.w * rs.w * (g.w - sg.w * inv_b - (((zz.w + b.w) - mu.w) * rs.w) * sx.w * inv_b);
    }
    *reinterpret_cast<float4*>(gz + i) = g;
  }
}

}  // namespace er

// Layout: 1024 reserved bytes, then the chunk partials [n_chunks][units][3].
extern "C" size_t er_dense_workspace_bytes(int64_t batch, int32_t units) {
  er::DenseShape s = er::dense_shape(batch > 0 ? batch : 1, units > 0 ? units : 1);
  er::VecShape v = er::vec_shape(batch > 0 ? batch : 1, units > 0 ? units : 1);
  const size_t scalar = (size_t)s.n_chunks * s.units * 3 * sizeof(float);
  const size_t vec = (size_t)v.n_chunks * (((size_t)v.units + 3) / 4 * 4) * 2 * sizeof(float);
  return 1024 + std::max(scalar, vec) + 256;
}

extern "C" int er_bias_bn_act_fwd(const float* z, const float* bias, const float* gamma,
                                  const float* beta, float* moving_mean, float* moving_var,
                                  int64_t batch, int32_t units, float eps, float momentum,
                                  int32_t training, int32_t relu, float* y, float* save_mean,
                                  float* save_rstd, void* ws, size_t ws_bytes, er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(z && y, "null argument");
  ER_REQUIRE(batch > 0 && units > 0, "bad shape");
  cudaStream_t st = as_stream(stream);
  if (!gamma) {
    bias_act_kernel<<<grid_for(batch * units, 256, 8), 256, 0, st>>>(z, bias, batch * units, units, relu, y);
    count_launches(1);
    ER_CUDA_LAUNCH_CHECK();
    return ER_OK;
  }
  ER_REQUIRE(beta && moving_mean && moving_var, "batch norm needs beta and moving statistics");
  DenseShape s = dense_shape(batch, units);
  dim3 grid((units + kColTile - 1) / kColTile, s.n_chunks);
  if (training) {
    ER_REQUIRE(save_mean && save_rstd, "training needs save_mean / save_rstd");
    if (!ws || ws_bytes < er_dense_workspace_bytes(batch, units))
      return fail(ER_ERR_WORKSPACE, "er_bias_bn_act_fwd: workspace too small");
    bn_stats_kernel<<<grid, 256, 0, st>>>(z, bias, s, reinterpret_cast<float*>(static_cast<char*>(ws) + 1024));
    count_launches(1);
  }
  bn_apply_kernel<<<grid, 256, 0, st>>>(z, bias, gamma, beta, moving_mean, moving_var, s, eps, momentum,
                                        training, relu,
                                        ws ? reinterpret_cast<const float*>(static_cast<char*>(ws) + 1024) : nullptr, y, save_mean,
                                        save_rstd);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_bn_act_apply(const float* z, const float* bias, const float* gamma, const float* beta,
                               const float* mean, const float* rstd, int64_t batch, int32_t units,
                               int32_t relu, float* y, er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(z && gamma && beta && mean && rstd && y, "null argument");
  ER_REQUIRE(batch > 0 && units > 0, "bad shape");
  cudaStream_t st = as_stream(stream);
  auto al = [](const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; };
  const int64_t total = batch * units;
  if (units % 4 == 0 && al(z) && al(y) && al(gamma) && al(beta) && al(mean) && al(rstd) && (!bias || al(bias))) {
    launch_pdl(bn_act_apply_vec_kernel, dim3(grid_for(total / 4, 256, 8)), dim3(256), 0, st,
               reinterpret_cast<const float4*>(z), bias, gamma, beta, mean, rstd, total / 4, (int)units, (int)relu,
               reinterpret_cast<float4*>(y));
  } else {
    bn_act_apply_kernel<<<grid_for(total, 256, 8), 256, 0, st>>>(z, bias, gamma, beta, mean, rstd, total, units,
                                                                 relu, y);
  }
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_bias_bn_act_bwd(const float* z, const float* bias, const float* gamma,
                                  const float* y, const float* gy, const float* save_mean,
                                  const float* save_rstd, int64_t batch, int32_t units,
                                  int32_t relu, float* gz, float* gbias, float* ggamma,
                                  float* gbeta, void* ws, size_t ws_bytes, er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(z && y && gy && gz, "null argument");
  ER_REQUIRE(batch > 0 && units > 0, "bad shape");
  const int use_bn = gamma != nullptr;
  ER_REQUIRE(!use_bn || (save_mean && save_rstd), "batch norm backward needs the saved statistics");
  if (!ws || ws_bytes < er_dense_workspace_bytes(batch, units))
    return fail(ER_ERR_WORKSPACE, "er_bias_bn_act_bwd: workspace too small");
  cudaStream_t st = as_stream(stream);
  DenseShape s = dense_shape(batch, units);
  dim3 grid((units + kColTile - 1) / kColTile, s.n_chunks);
  float* part = reinterpret_cast<float*>(static_cast<char*>(ws) + 1024);
  auto al = [](const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; };
  if (units % 4 == 0 && al(z) && al(y) && al(gy) && al(gz) && (!bias || al(bias)) && (!gbias || al(gbias)) &&
      (!use_bn || (al(gamma) && al(save_mean) && al(save_rstd) && (!ggamma || al(ggamma)) && (!gbeta || al(gbeta))))) {
    VecShape v = vec_shape(batch, units);
    dim3 vgrid((units + kVecCols - 1) / kVecCols, v.n_chunks);
    launch_pdl(bn_bwd_stats_vec_kernel<false>, vgrid, dim3(256), 0, st, z, bias, (const float*)nullptr,
               (const float*)nullptr, y, gy, save_mean, save_rstd, v, (int)relu, use_bn, part);
    launch_pdl(bn_bwd_apply_vec_kernel<false>, vgrid, dim3(256), 0, st, z, bias, gamma, (const float*)nullptr, y,
               gy, save_mean, save_rstd, v, (int)relu, use_bn, (const float*)part, gz, gbias, ggamma, gbeta);
    count_launches(2);
    ER_CUDA_LAUNCH_CHECK();
    return ER_OK;
  }
  bn_bwd_stats_kernel<<<grid, 256, 0, st>>>(z, bias, y, gy, save_mean, save_rstd, s, relu, use_bn, part);
  bn_bwd_apply_kernel<<<grid, 256, 0, st>>>(z, bias, gamma, y, gy, save_mean, save_rstd, s, relu, use_bn,
                                            part, gz, gbias, ggamma, gbeta);
  count_launches(2);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_bn_relu_bwd(const float* z, const float* bias, const float* gamma, const float* beta,
                              const float* save_mean, const float* save_rstd, const float* gy, int64_t batch,
                              int32_t units, int32_t relu, float* gz, float* gbias, float* ggamma, float* gbeta,
                              void* ws, size_t ws_bytes, er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(z && gamma && beta && save_mean && save_rstd && gy && gz, "null argument");
  ER_REQUIRE(batch > 0 && units > 0, "bad shape");
  auto al = [](const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; };
  ER_REQUIRE(units % 4 == 0 && al(z) && al(gamma) && al(beta) && al(save_mean) && al(save_rstd) && al(gy) && al(gz) &&
                 (!bias || al(bias)) && (!gbias || al(gbias)) && (!ggamma || al(ggamma)) &&
                 (!gbeta || al(gbeta)),
             "er_bn_relu_bwd needs units % 4 == 0 and 16-byte aligned arrays");
  cudaStream_t st = as_stream(stream);
  VecShape v = vec_shape(batch, units);
  dim3 vgrid((units + kVecCols - 1) / kVecCols, v.n_chunks);
  if (!ws || ws_bytes < er_dense_workspace_bytes(batch, units))
    return fail(ER_ERR_WORKSPACE, "er_bn_relu_bwd: workspace too small");
  float* part = reinterpret_cast<float*>(static_cast<char*>(ws) + 1024);
  launch_pdl(bn_bwd_stats_vec_kernel<true>, vgrid, dim3(256), 0, st, z, bias, gamma, beta, (const float*)nullptr, gy,
             save_mean, save_rstd, v, (int)relu, 1, part);
  launch_pdl(bn_bwd_apply_vec_kernel<true>, vgrid, dim3(256), 0, st, z, bias, gamma, beta, (const float*)nullptr, gy,
             save_mean, save_rstd, v, (int)relu, 1, (const float*)part, gz, gbias, ggamma, gbeta);
  count_launches(2);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

// ---- dropout of DNN.__call__ (layers/dnn.py:77-82: tf.nn.dropout(x, keep_prob = 1 - ratio), training only) ----------
// y = x * keep_mask / keep.  The mask is a counter-based function of (seed, step counter, element index): the backward
// pass recomputes it instead of storing it, and the step counter is a DEVICE scalar, so a captured CUDA graph draws a
// new mask on every replay (the host bumps the counter with one tiny device add after the backward).  TensorFlow's
// own random stream cannot be reproduced; the contract is the distribution (Bernoulli(keep) per element, E[y] = x).
namespace er {
__device__ __forceinline__ uint32_t drop_bits(uint64_t seed, uint64_t ctr, uint64_t i) {
  uint64_t z = seed + ctr * 0x9E3779B97F4A7C15ull + i * 0xD1B54A32D192ED03ull;   // splitmix64 finaliser
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return (uint32_t)((z ^ (z >> 31)) >> 32);
}

__global__ void __launch_bounds__(256)
    dropout_kernel(const float* __restrict__ x, int64_t n, uint64_t keep_thresh, float inv_keep, uint64_t seed,
                   const int64_t* __restrict__ counter, float* __restrict__ y) {
  const uint64_t ctr = (uint64_t)*counter;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    y[i] = (uint64_t)drop_bits(seed, ctr, (uint64_t)i) < keep_thresh ? x[i] * inv_keep : 0.f;
}
}  // namespace er

extern "C" int er_dropout(const float* x, int64_t n, float rate, uint64_t seed, const int64_t* counter_dev, float* y,
                          er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(x && y && counter_dev, "null argument");
  ER_REQUIRE(n > 0 && rate >= 0.f && rate < 1.f, "rate must be in [0, 1)");
  // kept iff the 32-bit draw is below floor(keep * 2^32), compared in 64 bits: at rate 0 the threshold is 2^32 and
  // every draw, 0xffffffff included, keeps its element
  const double keep = 1.0 - (double)rate;
  const uint64_t thresh = (uint64_t)(keep * 4294967296.0);
  dropout_kernel<<<grid_for(n, 256, 8), 256, 0, as_stream(stream)>>>(x, n, thresh, (float)(1.0 / keep), seed, counter_dev, y);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

// ---- the non-relu activations of get_activation (utils/activation.py:66-118; DNN.__call__ layers/dnn.py:70-73, keras
// MLP layers/keras/blocks.py:82) --------------------------------------------------------------------------------------
// ReLU stays fused in the bias / batch-norm epilogue above; a layer configured with another stateless activation runs
// that epilogue in its linear form and this elementwise pass on top.  The backward pass recomputes the derivative from
// the pre-activation x (kept for the batch-norm backward anyway), in the branch conventions of TF's gradient kernels
// (EluGrad / SeluGrad / LeakyReluGrad take the negative branch for x < 0 resp. x <= 0).
namespace er {
template <int KIND>
__global__ void __launch_bounds__(256) act_fwd_kernel(const float* __restrict__ x, int64_t n, float* __restrict__ y) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    y[i] = act_value<KIND>(x[i]);
}

template <int KIND>
__global__ void __launch_bounds__(256)
    act_bwd_kernel(const float* __restrict__ x, const float* __restrict__ gy, int64_t n, float* __restrict__ gx) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    gx[i] = gy[i] * act_slope<KIND>(x[i]);
}

template <int KIND>
static void act_launch(const float* x, const float* gy, int64_t n, float* out, cudaStream_t st) {
  const int grid = grid_for(n, 256 * 4, 8);
  if (gy)
    act_bwd_kernel<KIND><<<grid, 256, 0, st>>>(x, gy, n, out);
  else
    act_fwd_kernel<KIND><<<grid, 256, 0, st>>>(x, n, out);
}

static int act_dispatch(const float* x, const float* gy, int64_t n, int kind, float* out, er_stream_t stream) {
  cudaStream_t st = as_stream(stream);
  switch (kind) {
    case ER_ACT_GELU: act_launch<ER_ACT_GELU>(x, gy, n, out, st); break;
    case ER_ACT_LEAKY_RELU: act_launch<ER_ACT_LEAKY_RELU>(x, gy, n, out, st); break;
    case ER_ACT_ELU: act_launch<ER_ACT_ELU>(x, gy, n, out, st); break;
    case ER_ACT_SELU: act_launch<ER_ACT_SELU>(x, gy, n, out, st); break;
    case ER_ACT_TANH: act_launch<ER_ACT_TANH>(x, gy, n, out, st); break;
    case ER_ACT_SWISH: act_launch<ER_ACT_SWISH>(x, gy, n, out, st); break;
    case ER_ACT_SIGMOID: act_launch<ER_ACT_SIGMOID>(x, gy, n, out, st); break;
    default: return fail(ER_ERR_INVALID_ARG, "er_act: unknown activation kind");
  }
  count_launches(1);
  return ER_OK;
}
}  // namespace er

namespace er {
__global__ void __launch_bounds__(256)
    dice_fwd_kernel(const float* __restrict__ x, const float* __restrict__ xn, const float* __restrict__ alpha,
                    int64_t n, int units, float* __restrict__ y) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    y[i] = dice_value(x[i], xn[i], alpha[i % units]);
}
__global__ void __launch_bounds__(256)
    dice_bwd_kernel(const float* __restrict__ x, const float* __restrict__ xn, const float* __restrict__ alpha,
                    const float* __restrict__ gy, int64_t n, int units, float* __restrict__ gx_direct,
                    float* __restrict__ gxn, float* __restrict__ galpha_terms) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    dice_grads(x[i], xn[i], alpha[i % units], gy[i], gx_direct + i, gxn + i, galpha_terms + i);
}
}  // namespace er

extern "C" int er_dice_fwd(const float* x, const float* xn, const float* alpha, int64_t batch, int32_t units, float* y,
                           er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(x && xn && alpha && y, "null argument");
  ER_REQUIRE(batch > 0 && units > 0, "bad shape");
  const int64_t n = batch * units;
  dice_fwd_kernel<<<grid_for(n, 256 * 4, 8), 256, 0, as_stream(stream)>>>(x, xn, alpha, n, (int)units, y);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_dice_bwd(const float* x, const float* xn, const float* alpha, const float* gy, int64_t batch,
                           int32_t units, float* gx_direct, float* gxn, float* galpha_terms, er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(x && xn && alpha && gy && gx_direct && gxn && galpha_terms, "null argument");
  ER_REQUIRE(batch > 0 && units > 0, "bad shape");
  const int64_t n = batch * units;
  dice_bwd_kernel<<<grid_for(n, 256 * 4, 8), 256, 0, as_stream(stream)>>>(x, xn, alpha, gy, n, (int)units, gx_direct, gxn,
                                                                        galpha_terms);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_act_fwd(const float* x, int64_t n, int kind, float* y, er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(x && y, "null argument");
  ER_REQUIRE(n > 0, "n must be positive");
  int rc = act_dispatch(x, nullptr, n, kind, y, stream);
  if (rc != ER_OK) return rc;
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_act_bwd(const float* x, const float* gy, int64_t n, int kind, float* gx, er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(x && gy && gx, "null argument");
  ER_REQUIRE(n > 0, "n must be positive");
  int rc = act_dispatch(x, gy, n, kind, gx, stream);
  if (rc != ER_OK) return rc;
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

// ---- dense optimizer: every dense parameter lives in ONE flat fp32 buffer (params, grads and
// optimizer state are flat arrays with the same segment table), so the whole dense update of
// optimize_loss -> opt.apply_gradients (compat/optimizers.py:413-416) is one launch:
//   g = grad + l2 * w          (kernel_regularizer = l2_regularizer(scale), layers/dnn.py:57-62)
//   adagrad: acc += g^2 ; w -= lr * g * rsqrt(acc)            (tf.train.AdagradOptimizer)
//   adam   : m = b1 m + (1-b1) g ; v = b2 v + (1-b2) g^2 ; w -= lr_t * m / (sqrt(v) + eps)
// reg_loss_out (optional) accumulates sum l2/2 * w^2 of the pre-update weights (reporting only).
namespace er {

// Work items are 256-element chunks of the segments, numbered across all segments (prefix of chunk
// counts built per CTA in shared memory, binary search per chunk): one wave covers every tensor, however
// small, without a grid dimension per tensor.
__global__ void __launch_bounds__(256)
    dense_apply_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ s0,
                       float* __restrict__ s1, const er_dense_seg_t* __restrict__ segs, int n_segs, er_opt_t opt,
                       const float* __restrict__ lr_dev, float* __restrict__ reg_loss_out) {
  er_pdl_wait();
  extern __shared__ int s_first[];   // [n_segs + 1] first chunk of every segment
  for (int i = threadIdx.x; i < n_segs; i += blockDim.x) s_first[i + 1] = (int)((segs[i].n + 255) >> 8);
  __syncthreads();
  if (threadIdx.x == 0) {   // exclusive prefix in shared memory (the loads above were issued in parallel)
    int acc = 0;
    for (int i = 0; i < n_segs; ++i) {
      const int c = s_first[i + 1];
      s_first[i] = acc;
      acc += c;
    }
    s_first[n_segs] = acc;
  }
  __syncthreads();
  const int n_chunks = s_first[n_segs];
  // step scalars: a device scalar (lr_dev: already the effective rate), or lr and Adam's beta powers from the
  // caller's hyper-parameter block (opt.hyper_dev) or else from the struct itself; Adam's lr_t is formed from
  // those here, the same way for both sources and as er_embedding_bwd / er_sparse_apply form it
  float lr0;
  if (lr_dev) {
    lr0 = *lr_dev;
  } else {
    const float* hy = opt.hyper_dev;
    lr0 = hy ? __ldg(hy + ER_HYPER_LR) : opt.lr;
    if (opt.kind == ER_OPT_LAZY_ADAM || opt.kind == ER_OPT_ADAM_ROWS)
      lr0 = adam_lr_t_of(lr0, hy ? __ldg(hy + ER_HYPER_BETA1_POWER) : opt.beta1_power,
                         hy ? __ldg(hy + ER_HYPER_BETA2_POWER) : opt.beta2_power);
  }
  float reg = 0.f;
  for (int ch = blockIdx.x; ch < n_chunks; ch += gridDim.x) {
    int lo = 0, hi = n_segs;   // s_first[lo] <= ch < s_first[hi]
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (s_first[mid] <= ch) lo = mid; else hi = mid;
    }
    const er_dense_seg_t seg = segs[lo];
    const float lr = lr0 * seg.lr_mult;
    const int64_t i = (int64_t)(ch - s_first[lo]) * 256 + threadIdx.x;
    if (i >= seg.n) continue;
    const int64_t j = seg.offset + i;
    float w = p[j];
    float gr = g[j] * opt.grad_scale;
    if (seg.l2 != 0.f) {
      reg += 0.5f * seg.l2 * w * w;
      gr += seg.l2 * w;
    }
    if (opt.kind == ER_OPT_ADAGRAD) {
      const float a = s0[j] + gr * gr;
      s0[j] = a;
      w -= lr * gr * __frsqrt_rn(a);
    } else if (opt.kind == ER_OPT_LAZY_ADAM || opt.kind == ER_OPT_ADAM_ROWS) {
      const float m = opt.beta1 * s0[j] + (1.0f - opt.beta1) * gr;
      const float v = opt.beta2 * s1[j] + (1.0f - opt.beta2) * gr * gr;
      s0[j] = m;
      s1[j] = v;
      w -= lr * m / (sqrtf(v) + opt.eps);
    } else if (opt.kind == ER_OPT_MOMENTUM) {   // ApplyMomentum: accum = accum * momentum + g ; var -= lr * accum
      const float a = __fadd_rn(__fmul_rn(s0[j], opt.beta1), gr);
      s0[j] = a;
      w -= lr * a;
    } else {
      w -= lr * gr;
    }
    p[j] = w;
  }
  if (reg_loss_out) {
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) reg += __shfl_xor_sync(0xffffffffu, reg, o);
    if ((threadIdx.x & 31) == 0 && reg != 0.f) atomicAdd(reg_loss_out, reg);
  }
}

}  // namespace er

extern "C" int er_dense_apply(float* params, const float* grads, float* state0, float* state1,
                              const er_dense_seg_t* segs, int32_t n_segs, int64_t max_seg_n,
                              const er_opt_t* opt, const float* lr_dev, float* reg_loss_out,
                              er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(params && grads && segs && opt, "null argument");
  ER_REQUIRE(n_segs > 0 && n_segs <= 8192 && max_seg_n > 0, "bad segment table");
  ER_REQUIRE(opt->kind == ER_OPT_SGD || state0, "optimizer state0 missing");
  ER_REQUIRE((opt->kind != ER_OPT_LAZY_ADAM && opt->kind != ER_OPT_ADAM_ROWS) || state1, "adam needs state1");
  // enough CTAs for the biggest tensor's chunks plus one per small tensor, capped at 8 waves
  const int grid = (int)min((int64_t)8 * kSmCount, ceil_div(max_seg_n, (int64_t)256) + n_segs);
  launch_pdl(dense_apply_kernel, dim3(grid), dim3(256), (size_t)(n_segs + 1) * sizeof(int), as_stream(stream), params,
             grads, state0, state1, segs, (int)n_segs, *opt, lr_dev, reg_loss_out);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}
