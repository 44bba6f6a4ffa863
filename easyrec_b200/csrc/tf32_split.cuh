// The 3xTF32 operand split of the dense GEMM, shared by the GEMM's in-kernel staging, the kernel that pre-splits the
// tower weights (gemm.cu) and the host-side check tests/native/tf32_split_host.cpp, so all three use one definition:
//
//     hi = x rounded to nearest onto 10 mantissa bits (a tf32 value),  lo = x - hi  (exact in fp32: hi + lo == x)
//
// for every finite x below the largest finite tf32 value plus half an ulp (|x| < 0x1.ffep127): the rounding of larger
// magnitudes carries into the exponent and gives hi = +-inf.
#pragma once
#include <stdint.h>
#include <string.h>

#ifdef __CUDACC__
#define ER_SPLIT_HD __host__ __device__ __forceinline__
#else
#define ER_SPLIT_HD inline
#endif

namespace er {

ER_SPLIT_HD void split_tf32(float x, float& hi, float& lo) {
#ifdef __CUDA_ARCH__
  hi = __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u);
#else
  uint32_t u;
  memcpy(&u, &x, 4);
  u = (u + 0x1000u) & 0xffffe000u;
  memcpy(&hi, &u, 4);
#endif
  lo = x - hi;
}

}  // namespace er
