// Calibration microbenchmark: how fast can the GPU serve random 64-byte (16 x fp32) row reads /
// read-modify-writes out of a table much larger than L2?  This is the practical ceiling for the
// gather (K2) and scatter-update (K7) kernels, next to the streaming-copy peak in
// MEASURED_PEAKS.json.   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/bin/mb_gather tools/microbench_gather.cu
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

__device__ __forceinline__ float4 ldnc(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}

// 4 lanes per row, UNROLL rows in flight per lane group; output written densely
template <int UNROLL>
__global__ void __launch_bounds__(256) gather_kernel(const float4* __restrict__ table, const int64_t* __restrict__ rows,
                                                     int64_t n, float4* __restrict__ out) {
  const int lane = threadIdx.x & 3;
  const int64_t n_groups = (int64_t)gridDim.x * 64;
  const int64_t g = (int64_t)blockIdx.x * 64 + (threadIdx.x >> 2);
  for (int64_t base = 0; base < n; base += n_groups * UNROLL) {
    int64_t r[UNROLL];
    float4 v[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      int64_t s = base + u * n_groups + g;
      r[u] = s < n ? rows[s] : -1;
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) v[u] = r[u] >= 0 ? ldnc(table + r[u] * 4 + lane) : make_float4(0, 0, 0, 0);
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      int64_t s = base + u * n_groups + g;
      if (s < n) out[s * 4 + lane] = v[u];
    }
  }
}

// one thread per row: 4 x 16 B loads of the same row in flight
template <int UNROLL>
__global__ void __launch_bounds__(256) gather_row_per_thread(const float4* __restrict__ table, const int64_t* __restrict__ rows,
                                                             int64_t n, float4* __restrict__ out) {
  const int64_t nt = (int64_t)gridDim.x * blockDim.x;
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (int64_t base = 0; base < n; base += nt * UNROLL) {
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      int64_t s = base + u * nt + t;
      if (s < n) {
        int64_t r = rows[s];
        float4 a = ldnc(table + r * 4), b = ldnc(table + r * 4 + 1), c = ldnc(table + r * 4 + 2), d = ldnc(table + r * 4 + 3);
        out[s * 4] = a; out[s * 4 + 1] = b; out[s * 4 + 2] = c; out[s * 4 + 3] = d;
      }
    }
  }
}

// read-modify-write of two 64 B rows (weight + accumulator), distinct rows
__global__ void __launch_bounds__(256) rmw_kernel(float4* __restrict__ table, float4* __restrict__ acc,
                                                  const int64_t* __restrict__ rows, int64_t n) {
  const int lane = threadIdx.x & 3;
  const int64_t g = (int64_t)blockIdx.x * 64 + (threadIdx.x >> 2);
  if (g >= n) return;
  const int64_t r = rows[g];
  float4 w = table[r * 4 + lane], a = acc[r * 4 + lane];
  a.x += 1e-3f; a.y += 1e-3f; a.z += 1e-3f; a.w += 1e-3f;
  w.x -= a.x * 1e-6f; w.y -= a.y * 1e-6f; w.z -= a.z * 1e-6f; w.w -= a.w * 1e-6f;
  table[r * 4 + lane] = w;
  acc[r * 4 + lane] = a;
}

// interleaved layout: one 128 B line per row = [w(16 floats) | acc(16 floats)]
__global__ void __launch_bounds__(256) rmw_interleaved_kernel(float4* __restrict__ tab2, const int64_t* __restrict__ rows, int64_t n) {
  const int lane = threadIdx.x & 3;
  const int64_t g = (int64_t)blockIdx.x * 64 + (threadIdx.x >> 2);
  if (g >= n) return;
  const int64_t r = rows[g];
  float4 w = tab2[r * 8 + lane], a = tab2[r * 8 + 4 + lane];
  a.x += 1e-3f; a.y += 1e-3f; a.z += 1e-3f; a.w += 1e-3f;
  w.x -= a.x * 1e-6f; w.y -= a.y * 1e-6f; w.z -= a.z * 1e-6f; w.w -= a.w * 1e-6f;
  tab2[r * 8 + lane] = w;
  tab2[r * 8 + 4 + lane] = a;
}
// gather the first 64 B of 128 B-strided rows
__global__ void __launch_bounds__(256) gather_strided_kernel(const float4* __restrict__ tab2, const int64_t* __restrict__ rows,
                                                             int64_t n, float4* __restrict__ out) {
  const int lane = threadIdx.x & 3;
  const int64_t g = (int64_t)blockIdx.x * 64 + (threadIdx.x >> 2);
  if (g >= n) return;
  out[g * 4 + lane] = ldnc(tab2 + rows[g] * 8 + lane);
}

__global__ void fill_rows(int64_t* rows, int64_t n, int64_t V, uint64_t seed) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t x = (uint64_t)i * 0x9E3779B97F4A7C15ULL + seed;
  x ^= x >> 31; x *= 0xBF58476D1CE4E5B9ULL; x ^= x >> 29; x *= 0x94D049BB133111EBULL; x ^= x >> 32;
  rows[i] = (int64_t)(x % (uint64_t)V);
}
__global__ void fill_perm(int64_t* rows, int64_t n, int64_t V) {  // distinct rows: i * stride mod V
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) rows[i] = (i * 7919LL * 64 + 12345) % V;
}
__global__ void flush_kernel(float* p, int64_t n, float v) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}

template <class F>
float time_it(F f, float* flush, int iters) {
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  float tot = 0;
  for (int it = 0; it < iters + 2; ++it) {
    flush_kernel<<<1184, 256>>>(flush, 64LL << 20, (float)it);
    cudaEventRecord(e0);
    f();
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    if (it >= 2) tot += ms;
  }
  return tot / iters;
}

int main(int argc, char** argv) {
  const int64_t V = 10000013;
  float4 *table, *acc, *out;
  int64_t* rows;
  float* flush;
  const int64_t nmax = 8LL << 20;
  CK(cudaMalloc(&table, V * 64));
  CK(cudaMalloc(&acc, V * 64));
  CK(cudaMalloc(&out, nmax * 64));
  CK(cudaMalloc(&rows, nmax * 8));
  CK(cudaMalloc(&flush, 256LL << 20));
  CK(cudaMemset(table, 0, V * 64));
  CK(cudaMemset(acc, 0, V * 64));
  const int64_t sizes[] = {319488, 1277952, 5111808};
  for (int64_t n : sizes) {
    fill_rows<<<(unsigned)((n + 255) / 256), 256>>>(rows, n, V / 2, 1234);
    CK(cudaDeviceSynchronize());
    const double bytes = (double)n * (8 + 64 + 64);
    auto report = [&](const char* name, float ms) {
      printf("n=%8lld %-28s %8.2f us  %7.1f GB/s (rows+ids+out)  %6.1f Mrows/s\n", (long long)n, name, ms * 1e3,
             bytes / (ms * 1e-3) / 1e9, n / (ms * 1e-3) / 1e6);
    };
    report("gather 4lanes unroll1", time_it([&] { gather_kernel<1><<<(unsigned)((n + 63) / 64), 256>>>(table, rows, n, out); }, flush, 10));
    report("gather 4lanes unroll4 1184", time_it([&] { gather_kernel<4><<<1184, 256>>>(table, rows, n, out); }, flush, 10));
    report("gather 4lanes unroll8 1184", time_it([&] { gather_kernel<8><<<1184, 256>>>(table, rows, n, out); }, flush, 10));
    report("gather 4lanes unroll4 full", time_it([&] { gather_kernel<4><<<(unsigned)((n / 4 + 63) / 64), 256>>>(table, rows, n, out); }, flush, 10));
    report("gather row/thread unroll1", time_it([&] { gather_row_per_thread<1><<<(unsigned)((n + 255) / 256), 256>>>(table, rows, n, out); }, flush, 10));
    report("gather row/thread unroll2", time_it([&] { gather_row_per_thread<2><<<(unsigned)((n / 2 + 255) / 256), 256>>>(table, rows, n, out); }, flush, 10));
    {
      float ms2 = time_it([&] { gather_strided_kernel<<<(unsigned)((n + 63) / 64), 256>>>(table, rows, n, out); }, flush, 10);
      report("gather 64B of 128B-stride rows", ms2);
    }
    fill_perm<<<(unsigned)((n + 255) / 256), 256>>>(rows, n, V / 2);
    CK(cudaDeviceSynchronize());
    {
      float ms2 = time_it([&] { rmw_interleaved_kernel<<<(unsigned)((n + 63) / 64), 256>>>(table, rows, n); }, flush, 10);
      printf("n=%8lld %-28s %8.2f us  %7.1f GB/s (1 line r+w + ids)  %6.1f Mrows/s\n", (long long)n, "rmw interleaved [w|acc] 128B", ms2 * 1e3,
             (double)n * (8 + 256) / (ms2 * 1e-3) / 1e9, n / (ms2 * 1e-3) / 1e6);
    }
    fill_perm<<<(unsigned)((n + 255) / 256), 256>>>(rows, n, V);
    CK(cudaDeviceSynchronize());
    float ms = time_it([&] { rmw_kernel<<<(unsigned)((n + 63) / 64), 256>>>(table, acc, rows, n); }, flush, 10);
    printf("n=%8lld %-28s %8.2f us  %7.1f GB/s (2 rows r+w + ids)  %6.1f Mrows/s\n", (long long)n, "rmw w+acc distinct rows", ms * 1e3,
           (double)n * (8 + 256) / (ms * 1e-3) / 1e9, n / (ms * 1e-3) / 1e6);
  }
  // streaming reference
  {
    const int64_t n = 64LL << 20;  // floats
    float ms = time_it([&] { flush_kernel<<<1184, 256>>>((float*)out, n, 1.f); }, flush, 5);
    printf("stream write 256 MB: %.2f us %.1f GB/s\n", ms * 1e3, n * 4.0 / (ms * 1e-3) / 1e9);
  }
  CK(cudaDeviceSynchronize());
  return 0;
}
