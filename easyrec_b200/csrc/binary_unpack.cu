// CriteoInput batches on the device: the reference's binary parts (input/criteo_binary_reader.py) hold, per sample, an
// int32 label, 13 float32 dense values and 26 uint32 categories, row-major.  The readers' batch form is feature-major
// int64 ids, the dense columns in the input layer's order and float labels.  One CTA takes a tile of rows: it stages
// the tile's category and dense rows in shared memory with coalesced loads, then writes, per id slot, the tile's run of
// contiguous int64 values, and per raw column its values.  A pure stream of ~424 B per sample: at the sizes of a
// training batch the launch, not HBM, is its cost.
#include "common.cuh"

namespace er {

constexpr int kUnpackRows = 128;
constexpr int kUnpackThreads = 256;
constexpr int kCatPitch = ER_CRITEO_N_CAT + 1;      // odd pitches: a warp reading one column hits 32 banks
constexpr int kDensePitch = ER_CRITEO_N_DENSE;

__global__ void __launch_bounds__(kUnpackThreads)
    binary_unpack_kernel(const int32_t* __restrict__ label, const float* __restrict__ dense,
                         const uint32_t* __restrict__ cat, int64_t batch, const int32_t* __restrict__ slot_cols,
                         int32_t n_slot, const int32_t* __restrict__ raw_cols, int32_t n_raw,
                         int64_t* __restrict__ sparse_fea, float* __restrict__ dense_fea, float* __restrict__ labels) {
  __shared__ uint32_t s_cat[kUnpackRows * kCatPitch];
  __shared__ float s_dense[kUnpackRows * kDensePitch];
  const int64_t row0 = (int64_t)blockIdx.x * kUnpackRows;
  const int rows = (int)(batch - row0 < kUnpackRows ? batch - row0 : kUnpackRows);
  if (n_slot > 0) {
    const uint32_t* src = cat + row0 * ER_CRITEO_N_CAT;
    for (int e = threadIdx.x; e < rows * ER_CRITEO_N_CAT; e += blockDim.x)
      s_cat[(e / ER_CRITEO_N_CAT) * kCatPitch + e % ER_CRITEO_N_CAT] = __ldg(src + e);
  }
  if (n_raw > 0) {
    const float* src = dense + row0 * ER_CRITEO_N_DENSE;
    for (int e = threadIdx.x; e < rows * ER_CRITEO_N_DENSE; e += blockDim.x) s_dense[e] = __ldg(src + e);
  }
  for (int r = threadIdx.x; r < rows; r += blockDim.x) labels[row0 + r] = (float)__ldg(label + row0 + r);
  __syncthreads();
  // slot s, row r -> sparse_fea[s * batch + row0 + r]: consecutive threads write consecutive int64 of one slot's run
  for (int i = threadIdx.x; i < n_slot * kUnpackRows; i += blockDim.x) {
    const int s = i / kUnpackRows, r = i % kUnpackRows;
    if (r < rows)   // uint32 bits read as int32, the reference's declared tf.int32 (criteo_input.py: output_types)
      sparse_fea[(int64_t)s * batch + row0 + r] = (int64_t)(int32_t)s_cat[r * kCatPitch + __ldg(slot_cols + s)];
  }
  for (int i = threadIdx.x; i < rows * n_raw; i += blockDim.x) {
    const int r = i / n_raw, j = i % n_raw;
    dense_fea[(row0 + r) * n_raw + j] = s_dense[r * kDensePitch + __ldg(raw_cols + j)];
  }
}

}  // namespace er

extern "C" int er_binary_unpack(const int32_t* label, const float* dense, const uint32_t* cat, int64_t batch,
                                const int32_t* slot_cols, int32_t n_slot, const int32_t* raw_cols, int32_t n_raw,
                                int64_t* sparse_fea, float* dense_fea, float* labels, er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(label && labels, "null label array");
  ER_REQUIRE(batch > 0, "batch must be positive");
  ER_REQUIRE(n_slot >= 0 && n_raw >= 0 && n_raw <= ER_CRITEO_N_DENSE, "n_slot must be >= 0 and n_raw in [0, 13]");
  ER_REQUIRE(n_slot == 0 || (cat && slot_cols && sparse_fea), "null category, slot map or sparse_fea array");
  ER_REQUIRE(n_raw == 0 || (dense && raw_cols && dense_fea), "null dense, raw-column map or dense_fea array");
  const int64_t grid = ceil_div(batch, kUnpackRows);
  ER_REQUIRE(grid <= 0x7fffffff, "batch too large");
  binary_unpack_kernel<<<(unsigned)grid, kUnpackThreads, 0, as_stream(stream)>>>(
      label, dense, cat, batch, slot_cols, n_slot, raw_cols, n_raw, sparse_fea, dense_fea, labels);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}
