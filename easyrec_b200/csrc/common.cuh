// Shared helpers for liber_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>

#include <string>

#include "er_b200.h"

namespace er {

void set_error(const std::string& msg);
void count_launches(int n);  // kernels enqueued by this library (er_launch_count)

inline int fail(int code, const std::string& msg) {
  set_error(msg);
  return code;
}

#define ER_REQUIRE(cond, msg)                                              \
  do {                                                                     \
    if (!(cond)) return ::er::fail(ER_ERR_INVALID_ARG, std::string(__func__) + ": " + (msg)); \
  } while (0)

#define ER_CUDA_LAUNCH_CHECK()                                             \
  do {                                                                     \
    cudaError_t e__ = cudaPeekAtLastError();                               \
    if (e__ != cudaSuccess) {                                              \
      cudaGetLastError();                                                  \
      return ::er::fail(ER_ERR_CUDA, std::string(__func__) + ": " + cudaGetErrorString(e__)); \
    }                                                                      \
  } while (0)

constexpr int kSmCount = 132;  // H100 SXM

__host__ __device__ inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

inline cudaStream_t as_stream(er_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

// Cap a 1-D grid: enough CTAs to cover `work_items` at `per_cta`, rounded so
// large problems run as whole waves of the 132 SMs (grid-stride loops inside).
inline int grid_for(int64_t work_items, int per_cta, int ctas_per_sm) {
  int64_t need = ceil_div(work_items, per_cta);
  int64_t wave = (int64_t)kSmCount * ctas_per_sm;
  if (need <= 0) return 1;
  if (need <= wave) return (int)need;
  return (int)wave;
}

// 16-byte streaming load / store that do not allocate in L1 (rows are touched
// once per launch; L2 keeps the hot Zipf head).
__device__ __forceinline__ float4 ld_row_f4(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream_f4(float4* p, const float4& v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x),
               "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

// ---- programmatic dependent launch (PDL) ----------------------------------------------------------
// The step is a chain of short kernels.  Launched with the programmatic-stream-serialization attribute, a
// kernel's CTAs may be scheduled while its predecessor is still draining: they run their prologue (barrier /
// shared-memory set-up, index math) and block in er_pdl_wait() until the predecessor has completed and its writes are
// visible - so correctness is exactly stream order, only launch latency and ramp-up overlap.  Every kernel
// launched through launch_pdl() calls er_pdl_wait() before its first global access and then lets its own
// successor start launching.  ER_PDL=0 in the environment turns the attribute off (plain launches).
__device__ __forceinline__ void er_pdl_wait() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
bool pdl_enabled();   // api.cu
template <typename... KArgs, typename... Args>
inline void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                       Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// lr * sqrt(1 - beta2_power) / (1 - beta1_power) in fp32, the order of the TF graph (adam_s.py:193);
// every operation correctly rounded so the host (adam_lr_t) and device values are the same float
__host__ __device__ __forceinline__ float adam_lr_t_of(float lr, float b1p, float b2p) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(__fmul_rn(lr, __fsqrt_rn(__fsub_rn(1.0f, b2p))), __fsub_rn(1.0f, b1p));
#else
  return lr * sqrtf(1.0f - b2p) / (1.0f - b1p);
#endif
}

// slot of a segment: largest f with slots[f].seg_begin <= s (slots sorted by seg_begin).
__device__ __forceinline__ int find_slot(const int32_t* __restrict__ seg_begins, int n_slots,
                                         int32_t s) {
  int lo = 0, hi = n_slots;  // invariant: seg_begins[lo] <= s < seg_begins[hi]
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (seg_begins[mid] <= s)
      lo = mid;
    else
      hi = mid;
  }
  return lo;
}

}  // namespace er
