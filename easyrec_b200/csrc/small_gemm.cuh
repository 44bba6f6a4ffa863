// Vector-sized GEMMs of the dense towers: C[M,N] = A(M,K) . B(K,N) (+ bias) when one of M, N, K is below 8 - the
// gate layers of MMoE (dense(x) -> [B, num_expert], layers/mmoe.py:66-72), their dX ([B, E] x [E, d]) and dW
// ([d, B] x [B, E], a reduction over the batch) - where a 128 x 128 tensor-core tile would be > 90 % padding.
// CUDA cores, fp32 FMA chains in index order (deterministic).  The cell function below is the whole arithmetic: the
// kernels (small_gemm.cu) only map threads to (output element, k-slice); tests/native/ compiles it for the CPU.
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define ER_SG_HD __host__ __device__ __forceinline__
#else
#define ER_SG_HD inline
#endif

namespace er {

struct SmallGemm {
  const float* a;   // A(i, k) = a[i * sa_i + k * sa_k]
  const float* b;   // B(k, j) = b[k * sb_k + j * sb_j]
  int64_t sa_i, sa_k, sb_k, sb_j;
  int64_t M, N, K;
  int64_t k_per_slice;   // K is cut into ceil(K / k_per_slice) slices (1 slice: no partials)
};

// how the K range is cut: outputs are few and K long (the dW form) -> slices of >= 64, about 2 waves of CTAs in all
ER_SG_HD int64_t small_gemm_slices(int64_t M, int64_t N, int64_t K) {
  const int64_t out_ctas = (M * N + 255) / 256;
  if (K < 512 || out_ctas >= 132) return 1;   // 132 = the H100 SXM's SM count
  int64_t s = (2 * 132 + out_ctas - 1) / out_ctas;
  const int64_t most = K / 64;
  if (s > most) s = most;
  return s < 1 ? 1 : s;
}

// partial sum of output element o = i * N + j over k-slice s, k ascending
ER_SG_HD float small_gemm_cell(const SmallGemm& g, int64_t o, int64_t s) {
  const int64_t i = o / g.N, j = o - i * g.N;
  const int64_t k0 = s * g.k_per_slice;
  int64_t k1 = k0 + g.k_per_slice;
  if (k1 > g.K) k1 = g.K;
  const float* pa = g.a + i * g.sa_i + k0 * g.sa_k;
  const float* pb = g.b + k0 * g.sb_k + j * g.sb_j;
  float acc = 0.f;
  for (int64_t k = k0; k < k1; ++k) {
    acc = fmaf(*pa, *pb, acc);
    pa += g.sa_k;
    pb += g.sb_k;
  }
  return acc;
}

// slices summed in slice order (+ bias[j])
ER_SG_HD float small_gemm_reduce(const float* part, int64_t n_out, int64_t n_slice, int64_t o, const float* bias,
                                 int64_t N) {
  float acc = part[o];
  for (int64_t s = 1; s < n_slice; ++s) acc += part[s * n_out + o];
  return bias ? acc + bias[o % N] : acc;
}

}  // namespace er
