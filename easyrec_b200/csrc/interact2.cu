// K4 DIN target attention, K5 DCN cross, MMoE mixture, DSSM similarity pieces.
// The matmuls inside these blocks (attention MLP, towers, U.I^T) are er_gemm calls (gemm.cu); what is
// here is everything around them, fused so that the [B,T,4D] / [B,E,H] intermediates are produced
// and consumed in one pass each.  One warp per sample: T <= a few hundred, D <= 128.
//   DIN   : layers/sequence_feature_layer.py:150-189, model/multi_tower_din.py:62-97
//   cross : model/dcn.py:32-45         x_{l+1} = x0 * (x_l . w) + b + x_l
//   MMoE  : layers/mmoe.py:53-83       sum_e softmax(gate)[e] * expert_e
//   DSSM  : model/dssm.py:64-71 (l2 normalise), model/match_model.py:50-69,213-234 (in-batch softmax)
#include "common.cuh"

namespace er {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- DIN: din_in[b,t,:] = [q, k, q-k, q*k] ------------------------------------------------
__global__ void __launch_bounds__(256)
    din_concat_fwd_kernel(const float* __restrict__ q, const float* __restrict__ keys, int64_t total,
                          int seq_len, int dim, float* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int d = (int)(i % dim);
    const int64_t bt = i / dim;
    const int64_t b = bt / seq_len;
    const float qv = q[b * dim + d], kv = keys[i];
    float* o = out + bt * 4 * dim + d;
    o[0] = qv;
    o[dim] = kv;
    o[2 * dim] = qv - kv;
    o[3 * dim] = qv * kv;
  }
}

// g_q[b,d] = sum_t (g0 + g2 + g3*k) ; g_k[b,t,d] (+)= g1 - g2 + g3*q      one thread per (b, d)
__global__ void __launch_bounds__(256)
    din_concat_bwd_kernel(const float* __restrict__ q, const float* __restrict__ keys,
                          const float* __restrict__ g, int64_t batch, int seq_len, int dim,
                          float* __restrict__ gq, float* __restrict__ gk, int accumulate_gk) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < batch * dim;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int d = (int)(i % dim);
    const int64_t b = i / dim;
    const float qv = q[i];
    float acc = 0.f;
    for (int t = 0; t < seq_len; ++t) {
      const int64_t bt = b * seq_len + t;
      const float* gg = g + bt * 4 * dim + d;
      const float kv = keys[bt * dim + d];
      const float g0 = gg[0], g1 = gg[dim], g2 = gg[2 * dim], g3 = gg[3 * dim];
      acc += g0 + g2 + g3 * kv;
      const float v = g1 - g2 + g3 * qv;
      if (accumulate_gk)
        gk[bt * dim + d] += v;
      else
        gk[bt * dim + d] = v;
    }
    gq[i] = acc;
  }
}

// scores masked at t >= len with -2^32+1, softmax over T, out[b,:] = sum_t p[b,t] * keys[b,t,:]
__global__ void __launch_bounds__(256)
    din_pool_fwd_kernel(const float* __restrict__ scores, const float* __restrict__ keys,
                        const int32_t* __restrict__ lens, int64_t batch, int seq_len, int dim,
                        float* __restrict__ probs, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= batch) return;
  const int len = lens ? lens[b] : seq_len;
  const float kPad = -4294967295.0f;  // -2**32 + 1
  float m = -INFINITY;
  for (int t = lane; t < seq_len; t += 32) m = fmaxf(m, t < len ? scores[b * seq_len + t] : kPad);
  m = warp_max(m);
  float s = 0.f;
  for (int t = lane; t < seq_len; t += 32) s += expf((t < len ? scores[b * seq_len + t] : kPad) - m);
  s = warp_sum(s);
  const float inv = 1.0f / s;
  for (int t = lane; t < seq_len; t += 32)
    probs[b * seq_len + t] = expf((t < len ? scores[b * seq_len + t] : kPad) - m) * inv;
  __syncwarp();
  for (int d = lane; d < dim; d += 32) {
    float acc = 0.f;
    for (int t = 0; t < seq_len; ++t) acc += probs[b * seq_len + t] * keys[(b * seq_len + t) * dim + d];
    out[b * dim + d] = acc;
  }
}

// dp[t] = gout . keys[t] ; g_score[t] = p[t] * (dp[t] - sum_t' p dp) (0 at masked t) ; g_keys (+)= p[t]*gout
__global__ void __launch_bounds__(256)
    din_pool_bwd_kernel(const float* __restrict__ probs, const float* __restrict__ keys,
                        const float* __restrict__ gout, const int32_t* __restrict__ lens, int64_t batch,
                        int seq_len, int dim, float* __restrict__ g_scores, float* __restrict__ g_keys,
                        int accumulate_gkeys) {
  const int lane = threadIdx.x & 31;
  const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= batch) return;
  const int len = lens ? lens[b] : seq_len;
  float dot_pd = 0.f;
  for (int t = 0; t < seq_len; ++t) {
    float dp = 0.f;
    for (int d = lane; d < dim; d += 32) dp += gout[b * dim + d] * keys[(b * seq_len + t) * dim + d];
    dp = warp_sum(dp);
    if (lane == 0) g_scores[b * seq_len + t] = dp;  // stash dp
    dot_pd += probs[b * seq_len + t] * dp;
  }
  __syncwarp();
  for (int t = lane; t < seq_len; t += 32) {
    const float p = probs[b * seq_len + t];
    const float v = p * (g_scores[b * seq_len + t] - dot_pd);
    g_scores[b * seq_len + t] = (t < len) ? v : 0.f;  // tf.where routes no gradient to padded scores
  }
  for (int t = 0; t < seq_len; ++t) {
    const float p = probs[b * seq_len + t];
    for (int d = lane; d < dim; d += 32) {
      const int64_t i = (b * seq_len + t) * dim + d;
      const float v = p * gout[b * dim + d];
      if (accumulate_gkeys)
        g_keys[i] += v;
      else
        g_keys[i] = v;
    }
  }
}

// attention_normalizer 'sigmoid' of the keras DIN block (layers/keras/din.py:57-60):
// p[b,t] = t < len ? sigmoid(scale * s[b,t]) : 0 (the masked score -2^32+1 gives exactly 0 in fp32 there),
// out[b,:] = sum_t p[b,t] * keys[b,t,:] in ascending t.  One warp per sample.
__global__ void __launch_bounds__(256)
    din_sigmoid_pool_fwd_kernel(const float* __restrict__ scores, const float* __restrict__ keys,
                                const int32_t* __restrict__ lens, int64_t batch, int seq_len, int dim,
                                float scale, float* __restrict__ probs, float* __restrict__ out) {
  er_pdl_wait();
  const int lane = threadIdx.x & 31;
  const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= batch) return;
  const int len = lens ? lens[b] : seq_len;
  for (int t = lane; t < seq_len; t += 32)
    probs[b * seq_len + t] = t < len ? 1.0f / (1.0f + expf(-scale * scores[b * seq_len + t])) : 0.f;
  __syncwarp();
  for (int d = lane; d < dim; d += 32) {
    float acc = 0.f;
    for (int t = 0; t < seq_len; ++t) acc += probs[b * seq_len + t] * keys[(b * seq_len + t) * dim + d];
    out[b * dim + d] = acc;
  }
}

// g_score[t] = t < len ? scale * p (1 - p) * (gout . keys[t]) : 0 ; g_keys[t,:] (+)= p[t] * gout
__global__ void __launch_bounds__(256)
    din_sigmoid_pool_bwd_kernel(const float* __restrict__ probs, const float* __restrict__ keys,
                                const float* __restrict__ gout, const int32_t* __restrict__ lens, int64_t batch,
                                int seq_len, int dim, float scale, float* __restrict__ g_scores,
                                float* __restrict__ g_keys, int accumulate_gkeys) {
  er_pdl_wait();
  const int lane = threadIdx.x & 31;
  const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= batch) return;
  const int len = lens ? lens[b] : seq_len;
  for (int t = 0; t < seq_len; ++t) {
    const float p = probs[b * seq_len + t];
    float dp = 0.f;
    for (int d = lane; d < dim; d += 32) {
      const int64_t i = (b * seq_len + t) * dim + d;
      const float g = gout[b * dim + d];
      dp += g * keys[i];
      const float v = p * g;
      if (accumulate_gkeys)
        g_keys[i] += v;
      else
        g_keys[i] = v;
    }
    dp = warp_sum(dp);
    if (lane == 0) g_scores[b * seq_len + t] = t < len ? scale * p * (1.0f - p) * dp : 0.f;
  }
}

// ---- DCN v1 cross layer ------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    cross_fwd_kernel(const float* __restrict__ x0, const float* __restrict__ xl, const float* __restrict__ w,
                     const float* __restrict__ bias, int64_t batch, int dim, float* __restrict__ out,
                     float* __restrict__ xw_out) {
  const int lane = threadIdx.x & 31;
  const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= batch) return;
  float acc = 0.f;
  for (int d = lane; d < dim; d += 32) acc += xl[b * dim + d] * w[d];
  acc = warp_sum(acc);
  if (lane == 0 && xw_out) xw_out[b] = acc;
  for (int d = lane; d < dim; d += 32) out[b * dim + d] = x0[b * dim + d] * acc + bias[d] + xl[b * dim + d];
}

// s[b] = sum_d gout*x0 ; gxl = gout + w*s ; gx0 (+)= gout*xw
__global__ void __launch_bounds__(256)
    cross_bwd_kernel(const float* __restrict__ x0, const float* __restrict__ w, const float* __restrict__ xw,
                     const float* __restrict__ gout, int64_t batch, int dim, float* __restrict__ gx0,
                     float* __restrict__ gxl, float* __restrict__ s_out, int accumulate_gx0) {
  const int lane = threadIdx.x & 31;
  const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= batch) return;
  float s = 0.f;
  for (int d = lane; d < dim; d += 32) s += gout[b * dim + d] * x0[b * dim + d];
  s = warp_sum(s);
  if (lane == 0) s_out[b] = s;
  const float xwb = xw[b];
  for (int d = lane; d < dim; d += 32) {
    const float g = gout[b * dim + d];
    gxl[b * dim + d] = g + w[d] * s;
    const float v = g * xwb;
    if (accumulate_gx0)
      gx0[b * dim + d] += v;
    else
      gx0[b * dim + d] = v;
  }
}

// column reductions over the batch, deterministic two-stage: part[chunk][col] then a tree of chunks
//   out0[col] = sum_b a[b,col] * (scale ? scale[b] : 1)     out1[col] = sum_b c[b,col] (optional)
__global__ void __launch_bounds__(256)
    colsum_partial_kernel(const float* __restrict__ a, const float* __restrict__ scale,
                          const float* __restrict__ c, int64_t batch, int dim, int rows_per_chunk,
                          float* __restrict__ part) {
  __shared__ float s0[8][32], s1[8][32];
  const int col = blockIdx.x * 32 + (threadIdx.x & 31);
  const int rl = threadIdx.x >> 5;
  const int64_t r0 = (int64_t)blockIdx.y * rows_per_chunk, r1 = min(batch, r0 + rows_per_chunk);
  float v0 = 0.f, v1 = 0.f;
  if (col < dim)
    for (int64_t r = r0 + rl; r < r1; r += 8) {
      v0 += a[r * dim + col] * (scale ? scale[r] : 1.f);
      if (c) v1 += c[r * dim + col];
    }
  s0[rl][threadIdx.x & 31] = v0;
  s1[rl][threadIdx.x & 31] = v1;
  __syncthreads();
  if (rl == 0 && col < dim) {
    for (int k = 1; k < 8; ++k) {
      v0 += s0[k][threadIdx.x];
      v1 += s1[k][threadIdx.x];
    }
    part[((int64_t)blockIdx.y * dim + col) * 2] = v0;
    part[((int64_t)blockIdx.y * dim + col) * 2 + 1] = v1;
  }
}
__global__ void __launch_bounds__(256)
    colsum_final_kernel(const float* __restrict__ part, int n_chunks, int dim, float* __restrict__ out0,
                        float* __restrict__ out1) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= dim) return;
  float v0 = 0.f, v1 = 0.f;
  for (int k = 0; k < n_chunks; ++k) {
    v0 += part[((int64_t)k * dim + col) * 2];
    v1 += part[((int64_t)k * dim + col) * 2 + 1];
  }
  out0[col] = v0;
  if (out1) out1[col] = v1;
}

// ---- MMoE mixture ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    mmoe_mix_fwd_kernel(const float* __restrict__ gate_logits, const float* __restrict__ experts,
                        int64_t batch, int n_expert, int dim, float* __restrict__ probs,
                        float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= batch) return;
  float m = -INFINITY;
  for (int e = lane; e < n_expert; e += 32) m = fmaxf(m, gate_logits[b * n_expert + e]);
  m = warp_max(m);
  float s = 0.f;
  for (int e = lane; e < n_expert; e += 32) s += expf(gate_logits[b * n_expert + e] - m);
  s = warp_sum(s);
  for (int e = lane; e < n_expert; e += 32)
    probs[b * n_expert + e] = expf(gate_logits[b * n_expert + e] - m) / s;
  __syncwarp();
  for (int d = lane; d < dim; d += 32) {
    float acc = 0.f;
    for (int e = 0; e < n_expert; ++e) acc += probs[b * n_expert + e] * experts[(b * n_expert + e) * dim + d];
    out[b * dim + d] = acc;
  }
}

__global__ void __launch_bounds__(256)
    mmoe_mix_bwd_kernel(const float* __restrict__ probs, const float* __restrict__ experts,
                        const float* __restrict__ gout, int64_t batch, int n_expert, int dim,
                        float* __restrict__ g_gate, float* __restrict__ g_experts, int accumulate_gexp) {
  const int lane = threadIdx.x & 31;
  const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= batch) return;
  float dot_pd = 0.f;
  for (int e = 0; e < n_expert; ++e) {
    float dp = 0.f;
    for (int d = lane; d < dim; d += 32) dp += gout[b * dim + d] * experts[(b * n_expert + e) * dim + d];
    dp = warp_sum(dp);
    if (lane == 0) g_gate[b * n_expert + e] = dp;
    dot_pd += probs[b * n_expert + e] * dp;
  }
  __syncwarp();
  for (int e = lane; e < n_expert; e += 32)
    g_gate[b * n_expert + e] = probs[b * n_expert + e] * (g_gate[b * n_expert + e] - dot_pd);
  for (int e = 0; e < n_expert; ++e) {
    const float p = probs[b * n_expert + e];
    for (int d = lane; d < dim; d += 32) {
      const int64_t i = (b * n_expert + e) * dim + d;
      const float v = p * gout[b * dim + d];
      if (accumulate_gexp)
        g_experts[i] += v;
      else
        g_experts[i] = v;
    }
  }
}

// ---- DSSM ------------------------------------------------------------------------------------
// tf.nn.l2_normalize(x, axis=-1): y = x * rsqrt(max(sum x^2, 1e-12))
// inv_norm of a row clamped by the epsilon: 1/sqrt(1e-12f) rounded to fp32.  The forward stores exactly this
// constant for clamped rows (not a runtime rsqrtf of 1e-12f, which may differ from it in the last bits), so the
// backward can tell clamped rows from inv_norm alone.
constexpr float kL2ClampInv = 1e6f;
__global__ void __launch_bounds__(256)
    l2norm_fwd_kernel(const float* __restrict__ x, int64_t batch, int dim, float* __restrict__ y,
                      float* __restrict__ inv_norm) {
  const int lane = threadIdx.x & 31;
  const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= batch) return;
  float s = 0.f;
  for (int d = lane; d < dim; d += 32) s += x[b * dim + d] * x[b * dim + d];
  s = warp_sum(s);
  const float inv = s >= 1e-12f ? rsqrtf(s) : kL2ClampInv;   // NaN sums take the clamp, as fmaxf did
  if (lane == 0) inv_norm[b] = inv;
  for (int d = lane; d < dim; d += 32) y[b * dim + d] = x[b * dim + d] * inv;
}
// gx = inv * (gy - y * (gy . y)) above the clamp.  Below it max(sum x^2, 1e-12) passes no gradient to the sum, so
// gx = gy * inv (TF's gradient of the clamped form).  Rows are told apart by inv == kL2ClampInv, which also takes
// rows whose sum lies at 1e-12f or a few ulp above it, where rsqrtf rounds to the same value (there the two
// formulas differ by ~|y|^2 ~ 1 and TF's own gradient is discontinuous).
__global__ void __launch_bounds__(256)
    l2norm_bwd_kernel(const float* __restrict__ y, const float* __restrict__ inv_norm,
                      const float* __restrict__ gy, int64_t batch, int dim, float* __restrict__ gx) {
  const int lane = threadIdx.x & 31;
  const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= batch) return;
  const float inv = inv_norm[b];
  if (inv == kL2ClampInv) {
    for (int d = lane; d < dim; d += 32) gx[b * dim + d] = gy[b * dim + d] * inv;
    return;
  }
  float dot = 0.f;
  for (int d = lane; d < dim; d += 32) dot += gy[b * dim + d] * y[b * dim + d];
  dot = warp_sum(dot);
  for (int d = lane; d < dim; d += 32) gx[b * dim + d] = inv * (gy[b * dim + d] - y[b * dim + d] * dot);
}

// in-batch softmax cross entropy over sim [B, N] (N >= B): duplicates of the positive item are masked
// with -1e32 (match_model.py:50-69); loss_b = -log(softmax(row b)[b] + 1e-12) * w_b;
// g_sim[b,:] = w_b * inv_wsum * (-(1/(p_bb+1e-12)) * p_bb * (onehot - p))
__global__ void __launch_bounds__(256)
    inbatch_softmax_ce_kernel(const float* __restrict__ sim, const int64_t* __restrict__ item_ids,
                              const float* __restrict__ weights, int64_t batch, int n_cols, float inv_wsum,
                              float* __restrict__ loss_rows, float* __restrict__ probs_diag,
                              float* __restrict__ g_sim) {
  const int lane = threadIdx.x & 31;
  const int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= batch) return;
  const float* row = sim + b * n_cols;
  const int64_t my_id = item_ids ? item_ids[b] : 0;
  float m = -INFINITY;
  for (int j = lane; j < n_cols; j += 32) {
    float v = row[j];
    if (item_ids && j < batch && j != b && item_ids[j] == my_id) v -= 1e32f;
    m = fmaxf(m, v);
  }
  m = warp_max(m);
  float s = 0.f;
  for (int j = lane; j < n_cols; j += 32) {
    float v = row[j];
    if (item_ids && j < batch && j != b && item_ids[j] == my_id) v -= 1e32f;
    s += expf(v - m);
  }
  s = warp_sum(s);
  const float pbb = expf(row[b] - m) / s;
  const float w = weights ? weights[b] : 1.f;
  if (lane == 0) {
    loss_rows[b] = -logf(pbb + 1e-12f) * w * inv_wsum;
    if (probs_diag) probs_diag[b] = pbb;
  }
  if (g_sim) {
    const float coef = -w * inv_wsum * pbb / (pbb + 1e-12f);
    for (int j = lane; j < n_cols; j += 32) {
      float v = row[j];
      if (item_ids && j < batch && j != b && item_ids[j] == my_id) v -= 1e32f;
      const float p = expf(v - m) / s;
      g_sim[b * n_cols + j] = coef * ((j == b ? 1.f : 0.f) - p);
    }
  }
}

inline int warps_grid(int64_t batch) { return (int)ceil_div(batch, (int64_t)8); }

}  // namespace er

using namespace er;

extern "C" int er_din_concat_fwd(const float* query, const float* keys, int64_t batch, int32_t seq_len,
                                 int32_t dim, float* din_in, er_stream_t stream) {
  ER_REQUIRE(query && keys && din_in, "null argument");
  ER_REQUIRE(batch > 0 && seq_len > 0 && dim > 0, "bad shape");
  const int64_t total = batch * seq_len * dim;
  din_concat_fwd_kernel<<<grid_for(total, 256, 8), 256, 0, as_stream(stream)>>>(query, keys, total, seq_len,
                                                                              dim, din_in);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_din_concat_bwd(const float* query, const float* keys, const float* g_din_in,
                                 int64_t batch, int32_t seq_len, int32_t dim, float* g_query,
                                 float* g_keys, int32_t accumulate_gkeys, er_stream_t stream) {
  ER_REQUIRE(query && keys && g_din_in && g_query && g_keys, "null argument");
  ER_REQUIRE(batch > 0 && seq_len > 0 && dim > 0, "bad shape");
  din_concat_bwd_kernel<<<grid_for(batch * dim, 256, 8), 256, 0, as_stream(stream)>>>(
      query, keys, g_din_in, batch, seq_len, dim, g_query, g_keys, accumulate_gkeys);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_din_pool_fwd(const float* scores, const float* keys, const int32_t* lens, int64_t batch,
                               int32_t seq_len, int32_t dim, float* probs, float* out,
                               er_stream_t stream) {
  ER_REQUIRE(scores && keys && probs && out, "null argument");
  ER_REQUIRE(batch > 0 && seq_len > 0 && dim > 0, "bad shape");
  din_pool_fwd_kernel<<<warps_grid(batch), 256, 0, as_stream(stream)>>>(scores, keys, lens, batch, seq_len,
                                                                       dim, probs, out);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_din_pool_bwd(const float* probs, const float* keys, const float* gout,
                               const int32_t* lens, int64_t batch, int32_t seq_len, int32_t dim,
                               float* g_scores, float* g_keys, int32_t accumulate_gkeys,
                               er_stream_t stream) {
  ER_REQUIRE(probs && keys && gout && g_scores && g_keys, "null argument");
  ER_REQUIRE(batch > 0 && seq_len > 0 && dim > 0, "bad shape");
  din_pool_bwd_kernel<<<warps_grid(batch), 256, 0, as_stream(stream)>>>(
      probs, keys, gout, lens, batch, seq_len, dim, g_scores, g_keys, accumulate_gkeys);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_din_sigmoid_pool_fwd(const float* scores, const float* keys, const int32_t* lens,
                                       int64_t batch, int32_t seq_len, int32_t dim, float scale, float* probs,
                                       float* out, er_stream_t stream) {
  ER_REQUIRE(scores && keys && probs && out, "null argument");
  ER_REQUIRE(batch > 0 && seq_len > 0 && dim > 0, "bad shape");
  launch_pdl(din_sigmoid_pool_fwd_kernel, dim3(warps_grid(batch)), dim3(256), 0, as_stream(stream), scores, keys,
             lens, batch, seq_len, dim, scale, probs, out);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_din_sigmoid_pool_bwd(const float* probs, const float* keys, const float* gout,
                                       const int32_t* lens, int64_t batch, int32_t seq_len, int32_t dim,
                                       float scale, float* g_scores, float* g_keys, int32_t accumulate_gkeys,
                                       er_stream_t stream) {
  ER_REQUIRE(probs && keys && gout && g_scores && g_keys, "null argument");
  ER_REQUIRE(batch > 0 && seq_len > 0 && dim > 0, "bad shape");
  launch_pdl(din_sigmoid_pool_bwd_kernel, dim3(warps_grid(batch)), dim3(256), 0, as_stream(stream), probs, keys,
             gout, lens, batch, seq_len, dim, scale, g_scores, g_keys, (int)accumulate_gkeys);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_cross_fwd(const float* x0, const float* xl, const float* w, const float* b,
                            int64_t batch, int32_t dim, float* out, float* xw_out, er_stream_t stream) {
  ER_REQUIRE(x0 && xl && w && b && out, "null argument");
  ER_REQUIRE(batch > 0 && dim > 0, "bad shape");
  cross_fwd_kernel<<<warps_grid(batch), 256, 0, as_stream(stream)>>>(x0, xl, w, b, batch, dim, out, xw_out);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" size_t er_cross_workspace_bytes(int64_t batch, int32_t dim) {
  const int64_t chunks = ceil_div(batch > 0 ? batch : 1, (int64_t)256);
  return (size_t)(chunks * dim * 2 + (batch > 0 ? batch : 1)) * sizeof(float) + 256;
}

extern "C" int er_cross_bwd(const float* x0, const float* xl, const float* w, const float* xw,
                            const float* gout, int64_t batch, int32_t dim, float* gx0, float* gxl,
                            float* gw, float* gb, int32_t accumulate_gx0, void* ws, size_t ws_bytes,
                            er_stream_t stream) {
  ER_REQUIRE(x0 && xl && w && xw && gout && gx0 && gxl && gw && gb, "null argument");
  ER_REQUIRE(batch > 0 && dim > 0, "bad shape");
  if (!ws || ws_bytes < er_cross_workspace_bytes(batch, dim))
    return fail(ER_ERR_WORKSPACE, "er_cross_bwd: workspace too small");
  cudaStream_t st = as_stream(stream);
  float* s_buf = reinterpret_cast<float*>(ws);
  float* part = s_buf + batch;
  cross_bwd_kernel<<<warps_grid(batch), 256, 0, st>>>(x0, w, xw, gout, batch, dim, gx0, gxl, s_buf,
                                                     accumulate_gx0);
  // chunks of 256 rows, or of a multiple of 256 when that would need more than 65535 chunks (the gridDim.y
  // limit); fewer chunks than er_cross_workspace_bytes counts, and a fixed order for a given batch
  const int64_t rows_per_chunk = 256 * ceil_div(ceil_div(batch, (int64_t)256), (int64_t)65535);
  const int chunks = (int)ceil_div(batch, rows_per_chunk);
  dim3 grid((dim + 31) / 32, chunks);
  colsum_partial_kernel<<<grid, 256, 0, st>>>(xl, s_buf, gout, batch, dim, (int)rows_per_chunk, part);
  colsum_final_kernel<<<(dim + 255) / 256, 256, 0, st>>>(part, chunks, dim, gw, gb);
  count_launches(3);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_mmoe_mix_fwd(const float* gate_logits, const float* experts, int64_t batch,
                               int32_t n_expert, int32_t dim, float* probs, float* out,
                               er_stream_t stream) {
  ER_REQUIRE(gate_logits && experts && probs && out, "null argument");
  ER_REQUIRE(batch > 0 && n_expert > 0 && dim > 0, "bad shape");
  mmoe_mix_fwd_kernel<<<warps_grid(batch), 256, 0, as_stream(stream)>>>(gate_logits, experts, batch, n_expert,
                                                                       dim, probs, out);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_mmoe_mix_bwd(const float* probs, const float* experts, const float* gout, int64_t batch,
                               int32_t n_expert, int32_t dim, float* g_gate_logits, float* g_experts,
                               int32_t accumulate_gexperts, er_stream_t stream) {
  ER_REQUIRE(probs && experts && gout && g_gate_logits && g_experts, "null argument");
  ER_REQUIRE(batch > 0 && n_expert > 0 && dim > 0, "bad shape");
  mmoe_mix_bwd_kernel<<<warps_grid(batch), 256, 0, as_stream(stream)>>>(
      probs, experts, gout, batch, n_expert, dim, g_gate_logits, g_experts, accumulate_gexperts);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_l2norm_fwd(const float* x, int64_t batch, int32_t dim, float* y, float* inv_norm,
                             er_stream_t stream) {
  ER_REQUIRE(x && y && inv_norm, "null argument");
  ER_REQUIRE(batch > 0 && dim > 0, "bad shape");
  l2norm_fwd_kernel<<<warps_grid(batch), 256, 0, as_stream(stream)>>>(x, batch, dim, y, inv_norm);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_l2norm_bwd(const float* y, const float* inv_norm, const float* gy, int64_t batch,
                             int32_t dim, float* gx, er_stream_t stream) {
  ER_REQUIRE(y && inv_norm && gy && gx, "null argument");
  ER_REQUIRE(batch > 0 && dim > 0, "bad shape");
  l2norm_bwd_kernel<<<warps_grid(batch), 256, 0, as_stream(stream)>>>(y, inv_norm, gy, batch, dim, gx);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_inbatch_softmax_ce(const float* sim, const int64_t* item_ids, const float* weights,
                                     int64_t batch, int32_t n_cols, float inv_wsum, float* loss_rows,
                                     float* probs_diag, float* g_sim, er_stream_t stream) {
  ER_REQUIRE(sim && loss_rows, "null argument");
  ER_REQUIRE(batch > 0 && n_cols >= batch, "bad shape");
  inbatch_softmax_ce_kernel<<<warps_grid(batch), 256, 0, as_stream(stream)>>>(
      sim, item_ids, weights, batch, n_cols, inv_wsum, loss_rows, probs_diag, g_sim);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

// ---- batched Gram matrices: DLRM / DotInteraction pairwise dot products -------------------------------------
// out[b, i, j] = sum_k x[b, i, k] * x[b, j, k]   (model/dlrm.py:52-61 einsum 'bne,bme->bnm';
// layers/keras/interaction.py:47-128).  n and d are small (tens): one thread per output element, the sample's
// [n, d] block is read through L1; sequential sums (deterministic, the order of a CPU loop).
namespace er {
__global__ void __launch_bounds__(256)
    gram_fwd_kernel(const float* __restrict__ x, int64_t batch, int n, int d, float* __restrict__ out) {
  const int64_t total = batch * n * n;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = t / (n * n);
    const int ij = (int)(t - b * n * n);
    const int i = ij / n, j = ij - i * n;
    const float* xi = x + (b * n + i) * d;
    const float* xj = x + (b * n + j) * d;
    float acc = 0.f;
    for (int k = 0; k < d; ++k) acc = __fadd_rn(acc, __fmul_rn(xi[k], xj[k]));
    out[t] = acc;
  }
}
// gx[b, i, k] = sum_j (g[b, i, j] + g[b, j, i]) * x[b, j, k]
__global__ void __launch_bounds__(256)
    gram_bwd_kernel(const float* __restrict__ x, const float* __restrict__ g, int64_t batch, int n, int d,
                    float* __restrict__ gx) {
  const int64_t total = batch * n * d;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = t / (n * d);
    const int ik = (int)(t - b * n * d);
    const int i = ik / d, k = ik - i * d;
    const float* gb = g + b * n * n;
    const float* xb = x + b * n * d;
    float acc = 0.f;
    for (int j = 0; j < n; ++j)
      acc = __fadd_rn(acc, __fmul_rn(__fadd_rn(gb[i * n + j], gb[j * n + i]), xb[j * d + k]));
    gx[t] = acc;
  }
}
}  // namespace er

extern "C" int er_gram_fwd(const float* x, int64_t batch, int32_t n, int32_t dim, float* out, er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(x && out, "null argument");
  ER_REQUIRE(batch > 0 && n > 0 && dim > 0 && n <= 4096, "bad shape");
  gram_fwd_kernel<<<grid_for(batch * n * n, 256, 8), 256, 0, as_stream(stream)>>>(x, batch, n, dim, out);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_gram_bwd(const float* x, const float* g, int64_t batch, int32_t n, int32_t dim, float* gx,
                           er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(x && g && gx, "null argument");
  ER_REQUIRE(batch > 0 && n > 0 && dim > 0 && n <= 4096, "bad shape");
  gram_bwd_kernel<<<grid_for(batch * n * dim, 256, 8), 256, 0, as_stream(stream)>>>(x, g, batch, n, dim, gx);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}
