// TEST INFRASTRUCTURE: compiles easyrec_b200/csrc/tf32_split.cuh - the split the GEMM and the plane kernel are built
// from - with a plain C++ compiler, so the CPU suite checks the 3xTF32 operand split where no GPU is present.
#include "tf32_split.cuh"

extern "C" void host_split_tf32(const float* x, long n, float* hi, float* lo) {
  for (long i = 0; i < n; ++i) er::split_tf32(x[i], hi[i], lo[i]);
}
