// Elementwise formulas shared by the kernels and by the host-side check tests/native/elementwise_host.cpp: the SAME
// source is compiled for the device (dense.cu, metrics.cu) and, with a plain C++ compiler, for the CPU tests - so the
// formulas are checked on the CPU as well (the launches themselves are GPU tests).
#pragma once
#include <math.h>
#include <stdint.h>

#include "er_b200.h"

#ifdef __CUDACC__
#define ER_HD __host__ __device__ __forceinline__
#else
#define ER_HD inline
#endif

namespace er {

// ---- the stateless non-relu activations of get_activation (utils/activation.py:66-118) ---------------------------
// value and derivative from the pre-activation x, in the branch conventions of TF's gradient kernels (EluGrad / SeluGrad
// take the negative branch for x < 0, LeakyReluGrad for x <= 0).
template <int KIND>
ER_HD float act_value(float x) {
  if (KIND == ER_ACT_GELU) {   // x * 0.5 * (1 + tanh(sqrt(2/pi) * (x + 0.044715 x^3)))  (activation.py:46-60)
    const float u = 0.7978845608028654f * (x + 0.044715f * (x * x * x));
    return x * (0.5f * (1.0f + tanhf(u)));
  }
  if (KIND == ER_ACT_LEAKY_RELU) return fmaxf(0.2f * x, x);              // tf.nn.leaky_relu, alpha 0.2
  if (KIND == ER_ACT_ELU) return x < 0.f ? expm1f(x) : x;
  if (KIND == ER_ACT_SELU) return x < 0.f ? 1.7580993408473768f * expm1f(x) : 1.0507009873554805f * x;
  if (KIND == ER_ACT_TANH) return tanhf(x);
  if (KIND == ER_ACT_SWISH) return x / (1.0f + expf(-x));                 // x * sigmoid(x)
  return 1.0f / (1.0f + expf(-x));                                        // ER_ACT_SIGMOID
}

template <int KIND>
ER_HD float act_slope(float x) {
  if (KIND == ER_ACT_GELU) {
    const float c = 0.7978845608028654f;
    const float t = tanhf(c * (x + 0.044715f * (x * x * x)));
    const float sech2 = 1.0f - t * t;
    // once tanh saturates the second term is 0 (0 * x keeps its sign, and NaN at x = +-inf); without the branch
    // 1 + 0.134 x^2 overflows for |x| > 5e19 and the product 0 * inf turns a slope of 1 or 0 into NaN
    return 0.5f * (1.0f + t) + (sech2 == 0.f ? 0.f * x : 0.5f * x * sech2 * c * (1.0f + 3.0f * 0.044715f * x * x));
  }
  if (KIND == ER_ACT_LEAKY_RELU) return x > 0.f ? 1.0f : 0.2f;
  if (KIND == ER_ACT_ELU) return x < 0.f ? expf(x) : 1.0f;
  if (KIND == ER_ACT_SELU) return x < 0.f ? 1.7580993408473768f * expf(x) : 1.0507009873554805f;
  if (KIND == ER_ACT_TANH) {
    const float t = tanhf(x);
    return 1.0f - t * t;
  }
  const float s = 1.0f / (1.0f + expf(-x));
  if (KIND == ER_ACT_SWISH) return s * (1.0f + x * (1.0f - s));
  return s * (1.0f - s);
}


// ---- batch norm of a dense layer, before its relu: h = ((z + b) - mean) * rstd * gamma + beta ----------------------
// Every kernel that forms h (the forward apply, and the backward passes that recompute the relu mask h > 0 from z instead
// of reading y) calls this one function, with each rounding spelled out: the mask is then exactly y > 0.  The order is
// the one nvcc contracted the expression to before (add, sub, mul, then one fma), so y keeps its bits.
ER_HD float bn_pre_act(float z, float b, float mean, float rstd, float gamma, float beta) {
#ifdef __CUDA_ARCH__
  return __fmaf_rn(__fmul_rn(__fsub_rn(__fadd_rn(z, b), mean), rstd), gamma, beta);
#else
  return fmaf(((z + b) - mean) * rstd, gamma, beta);
#endif
}

// ---- dice (utils/activation.py:13-43, layers/keras/activation.py:24-73): the data-adaptive activation of DIN ------------
// p = sigmoid(xn), xn = batch_norm(x) without centre / scale (epsilon 1e-9);  y = alpha * (1 - p) * x + p * x.
// The normalisation itself runs on the batch-norm kernels; these are the gate and its three gradient terms.
ER_HD float dice_value(float x, float xn, float alpha) {
  const float p = 1.0f / (1.0f + expf(-xn));
  return alpha * (1.0f - p) * x + p * x;
}
// gx_direct: through the explicit x factors; gxn: into the normalised input (continues through the batch-norm
// backward); galpha: this element's term of d/d alpha[c] (summed over the rows by the caller)
ER_HD void dice_grads(float x, float xn, float alpha, float gy, float* gx_direct, float* gxn, float* galpha) {
  const float p = 1.0f / (1.0f + expf(-xn));
  *gx_direct = gy * (alpha * (1.0f - p) + p);
  *gxn = gy * x * (1.0f - alpha) * p * (1.0f - p);
  *galpha = gy * x * (1.0f - p);
}

// ---- tf.metrics.auc (model/rank_model.py:360-373) -------------------------------------------------------------------
// bin of a prediction = number of thresholds strictly below it (math_ops.greater(pred, thr)); thr ascending; a NaN
// prediction exceeds none.
ER_HD int auc_bin(const float* thr, int n_thr, float p) {
  int lo = 0, hi = n_thr;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (thr[mid] < p)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo;
}
// tf.to_int64(label) then cast to bool (rank_model.py:361, metrics_impl.auc): positive = truncated label != 0
ER_HD bool auc_positive(float label) { return (long long)label != 0; }

}  // namespace er
