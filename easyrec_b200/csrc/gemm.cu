// Dense-layer GEMM of the interaction stage on the Hopper tensor cores (wgmma), fp32 in / fp32 out with
// "3xTF32" operand splitting so logits stay within the 1e-4 budget of an fp32 CPU run:
//
//     x = hi + lo,  hi = tf32-rounded x,  lo = x - hi  (exact in fp32)
//     A.B ~= Alo.Bhi + Ahi.Blo + Ahi.Bhi      (three wgmma ... .tf32 per k-step, fp32 accumulate)
//
// Replaces the library SGEMMs of layers/dnn.py:50-87 (tf.layers.dense forward) and of its gradient
// (dX = dY.W^T, dW = X^T.dY) with one kernel that reads the operands *as they lie* in HBM.  wgmma takes
// 32-bit operands from shared memory only K-major, so every operand tile is staged as a K-major
// SWIZZLE_128B tile (128 rows of M or N x 32 k = 128 B per row, 16 B chunk ^= row % 8):
//   - an operand whose K index is contiguous (activations in forward/dX, W[in,out] in dX) is stored with
//     16 B vector stores, 8 threads per row;
//   - an operand whose M/N index is contiguous (W[in,out] in forward, X and dY in dW) is transposed on its
//     way into shared memory: a thread loads a 4 (k) x 4 (M/N) block as four 16 B rows (a warp reads 4 k-rows
//     x 128 contiguous bytes), transposes it in registers and stores 4 k of each M/N row with one 16 B store
//     per plane, as the K-major path does;
// so no transposed copy of any matrix is ever made.
//
// CTA = 128x128 output tile (one k-slice of it under split-K), 2 warpgroups:
//   - every thread is a producer: global -> registers -> hi/lo split -> swizzled st.shared into a 3-stage ring,
//     with kPrefetch k-blocks of loads in flight per thread;
//   - warpgroup g issues the wgmma's of output rows [64g, 64g+64) asynchronously and keeps one k-block of them
//     in flight while the CTA stages the next one (wait_group 1 with 3 stages: a stage is rewritten only after
//     both warpgroups have retired the wgmma's that read it);
//   - accumulators in registers: one for Ahi.Bhi and one for the two cross terms (the tensor core truncates
//     the fp32 accumulator on every accumulate: keeping the small terms apart brings the error down to an
//     fp32 SGEMM's);
//   - epilogue: both accumulators -> add -> shared-memory tile -> 512 B coalesced row stores (+ bias);
//     optionally the batch-norm statistics of the output columns (per-half shifted sums -> per-tile Welford ->
//     the last CTA of a column tile merges the tiles in order).
// The MMA width NM (16/32/64/128 columns) is a template parameter picked from N, so narrow layers do not pay
// for 128 columns of tensor-core work.
// Split-K partials are reduced by a second kernel in a fixed order: results are run-to-run deterministic.
// The kernel is launched with programmatic dependent launch: its prologue overlaps the previous kernel's drain.
//
// Pre-split B (er_gemm_planes): the dense towers' weights change once per step but every 128-row tile of a forward or
// dX GEMM would split (and, in forward, transpose) the same weight tiles again.  er_gemm_split_planes writes each
// weight once per step as hi / lo planes in the exact K-major SWIZZLE_128B byte order of a B stage, zero-padded to
// whole tiles ([row tile][k-block][NM rows][32 k]); the GEMM then fills a stage's B half with two bulk asynchronous
// copies (cp.async.bulk, completed on the stage's mbarrier) issued by one thread, and the threads only stage A.  The
// planes hold the bits the in-kernel split produces and the wgmma sequence is unchanged: results are bit-identical.
#include <algorithm>

#include "common.cuh"
#include "tf32_split.cuh"

namespace er {
namespace gemm {

constexpr int BM = 128, BN = 128, BK = 32;
constexpr int kStages = 3;
constexpr int kPrefetch = 2;      // k-blocks of global loads in flight per thread
constexpr int kPrefetchPre = 3;   // the same with a pre-split B (only A goes through registers)
constexpr int kThreads = 256;     // 2 warpgroups
constexpr int kTileBytes = 128 * 128;          // 128 rows x 128 B
constexpr int kStageBytes = 4 * kTileBytes;    // A hi, A lo, B hi, B lo
constexpr int kOutPitch = BN + 8;              // floats per row of the staged output tile (conflict-free float2)
constexpr int kStatFloats = 768;               // per-half Welford partials [2][128][3]; reused by the final merge
constexpr int kSmemBytes = kStages * kStageBytes + 1024 /* align slack */ + kStatFloats * 4 + 16 + kStages * 8;
static_assert(BM * kOutPitch * 4 <= kStages * kStageBytes, "output tile must fit in the stage ring");

struct Args {
  const float* A;
  const float* B;
  float* C;
  const float* bias;
  float* partials;
  long long lda, ldb, ldc;
  int M, N, K;
  int a_mn, b_mn;      // 1: the M (resp. N) index is the contiguous one in memory
  // pre-split B planes (er_gemm_planes): hi / lo, plane_tile_floats(N, K) floats per 128-row tile; B is unused
  const float* b_hi;
  const float* b_lo;
  long long b_tile_floats;
  int k_per_slice;     // multiple of BK
  int n_slices;
  // batch-norm statistics of the output columns (training forward of a dense+BN layer), optional
  float* bn_part;            // [m_tiles][N][3] Welford (n, mean, M2) per 128-row tile
  unsigned int* bn_counter;  // [n_tiles], zero on entry, left zero
  er_bn_stats_t bn;
};

// MMA width of an N-column output (= rows of its B operand): the narrowest of 16/32/64/128 that covers N; wider
// outputs are cut into 128-column tiles.
__host__ __device__ constexpr int mma_width(long long n) { return n > 64 ? 128 : n > 32 ? 64 : n > 16 ? 32 : 16; }
// floats of one 128-row tile of a pre-split plane of a [rows x K] K-major operand: ceil(K / BK) k-blocks of NM x BK
__host__ __device__ constexpr long long plane_tile_floats(long long rows, long long k) {
  return (k + BK - 1) / BK * mma_width(rows) * BK;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n.reg .pred p;\nWAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@!p bra WAIT_%=;\n}\n" ::"r"(bar), "r"(parity) : "memory");
}
// global -> shared bulk copy (bytes % 16 == 0, both ends 16 B aligned), completing `bytes` transactions on bar
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// wgmma shared-memory matrix descriptor of a K-major SWIZZLE_128B tile: 8-row groups 1024 B apart (SBO),
// LBO unused; a k-step of 8 tf32 moves the start address by 32 B inside the swizzle atom.
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3fff);
  d |= (uint64_t)1 << 16;                       // LBO (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;             // SBO
  d |= (uint64_t)1 << 62;                       // SWIZZLE_128B
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator accesses across the asynchronous wgmma's
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] += A[64 x 8] . B[N x 8]^T, both K-major in shared memory; d has N / 2 registers per thread.
__device__ __forceinline__ void wgmma_tf32(float (&d)[8], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7"
      "}, %8, %9, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(da), "l"(db), "r"(1));
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[16], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
      "}, %16, %17, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(1));
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, %32, %33, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(1));
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(1));
}

__device__ __forceinline__ float4 mask_chunk(float4 v, int nvalid) {
  if (nvalid < 4) {
    if (nvalid < 1) v.x = 0.f;
    if (nvalid < 2) v.y = 0.f;
    if (nvalid < 3) v.z = 0.f;
    v.w = 0.f;
  }
  return v;
}

// Which 4 elements thread (warp, lane) loads in pass j (0..3) of a k-block, relative to the tile origin:
//   K-major : row r = lane/8 + 4*warp + 32*j (M/N), k = 4*(lane%8) .. +3
//   MN-major: the thread owns a 4 (k) x 4 (M/N) block and pass j loads its k row j:
//             k = 4*kq + j, M/N = 4*mq .. +3,  kq = 4*(warp%2) + (lane/2)%4,  mq = 8*(warp/2) + 2*(lane/8) + lane%2
// A warp's MN-major load reads 4 k rows x 128 contiguous bytes.  Rows past K or M/N are not loaded (predicated,
// destination zeroed); the partial chunk at the K (K-major) or M/N (MN-major) edge is cleared by mask_chunk when
// the registers are staged.
struct Pos {
  int mn, k;   // first element's tile-relative M/N row and k column
};
__device__ __forceinline__ Pos pos_of(int mn_major, int warp, int lane, int j) {
  if (!mn_major) return Pos{(lane >> 3) + 4 * warp + 32 * j, 4 * (lane & 7)};
  const int kq = 4 * (warp & 1) + ((lane >> 1) & 3), mq = 8 * (warp >> 1) + 2 * (lane >> 3) + (lane & 1);
  return Pos{4 * mq, 4 * kq + j};
}
__device__ __forceinline__ float4 load_pos(const float* __restrict__ P, long long ld, int mn_major, Pos p,
                                           int mn0, int mn_end, int k0, int k_end) {
  const int mn = mn0 + p.mn, k = k0 + p.k;
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (!mn_major) {
    if (mn < mn_end && k < k_end) v = __ldg(reinterpret_cast<const float4*>(P + (long long)mn * ld + k));
  } else {
    if (k < k_end && mn < mn_end) v = __ldg(reinterpret_cast<const float4*>(P + (long long)k * ld + mn));
  }
  return v;   // pitch % 4 == 0 and the first element is valid: the 16 B lie inside the row
}
// byte offset of tile element (row, k) in a K-major SWIZZLE_128B tile
__device__ __forceinline__ uint32_t swz(int row, int k) {
  return (uint32_t)row * 128u + (uint32_t)((((k >> 2) ^ (row & 7)) << 4) + ((k & 3) << 2));
}
// hi / lo of 4 elements of tile row `row`, k = k4 .. k4+3, into the tile pair at `hi_tile` (lo tile kTileBytes
// further)
__device__ __forceinline__ void store_chunk(uint32_t hi_tile, int row, int k4, float4 v) {
  float4 hi, lo;
  split_tf32(v.x, hi.x, lo.x); split_tf32(v.y, hi.y, lo.y);
  split_tf32(v.z, hi.z, lo.z); split_tf32(v.w, hi.w, lo.w);
  const uint32_t o = hi_tile + swz(row, k4);
  asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(o), "f"(hi.x), "f"(hi.y), "f"(hi.z), "f"(hi.w) : "memory");
  asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(o + kTileBytes), "f"(lo.x), "f"(lo.y), "f"(lo.z), "f"(lo.w) : "memory");
}
// One thread's share of a k-block (the 4 passes `v`, loaded at `p`) into the tile pair at `hi_tile`.  Tile rows at
// or past `rows` are never read by the tensor core and are not written.  An MN-major block is transposed in
// registers, so each of its 4 M/N rows takes one 16 B store of 4 consecutive k per plane.  In a quarter-warp (8
// lanes) those stores hit rows 4*mq + e with mq%2 = 0, 1 and k chunks kq = 4 consecutive values: under the 128 B
// swizzle the 8 lanes land in 8 different 16 B chunk columns, i.e. in all 32 banks once (no conflict).
__device__ __forceinline__ void store_block(uint32_t hi_tile, int mn_major, const Pos (&p)[4], const float4 (&v)[4],
                                            int rows, int mn0, int mn_end, int k0, int k_end) {
  if (!mn_major) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (p[j].mn < rows) store_chunk(hi_tile, p[j].mn, p[j].k, mask_chunk(v[j], k_end - (k0 + p[j].k)));
    return;
  }
  if (p[0].mn >= rows) return;
  const int nvalid = mn_end - (mn0 + p[0].mn);
  float4 x[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) x[j] = mask_chunk(v[j], nvalid);
  store_chunk(hi_tile, p[0].mn + 0, p[0].k, make_float4(x[0].x, x[1].x, x[2].x, x[3].x));
  store_chunk(hi_tile, p[0].mn + 1, p[0].k, make_float4(x[0].y, x[1].y, x[2].y, x[3].y));
  store_chunk(hi_tile, p[0].mn + 2, p[0].k, make_float4(x[0].z, x[1].z, x[2].z, x[3].z));
  store_chunk(hi_tile, p[0].mn + 3, p[0].k, make_float4(x[0].w, x[1].w, x[2].w, x[3].w));
}

struct Welford {
  float n, mean, m2;
};
__device__ __forceinline__ void wf_merge(Welford& a, const Welford& b) {   // Chan et al., fixed order
  if (b.n == 0.f) return;
  const float n = a.n + b.n;
  const float d = b.mean - a.mean;
  a.mean += d * (b.n / n);
  a.m2 += b.m2 + d * d * (a.n * b.n / n);
  a.n = n;
}

template <int NM, bool kPreB>
__global__ void __launch_bounds__(kThreads, 1) gemm_tf32x3_kernel(Args a) {
  constexpr int R = NM / 2;   // accumulator registers per thread
  constexpr int kPf = kPreB ? kPrefetchPre : kPrefetch;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_u32 = smem_u32(smem_raw);
  const uint32_t smem_base = (raw_u32 + 1023u) & ~1023u;   // SWIZZLE_128B atoms: 1024 B aligned
  uint8_t* base_ptr = smem_raw + (smem_base - raw_u32);
  float* s_stats = reinterpret_cast<float*>(base_ptr + kStages * kStageBytes);
  int* s_flag = reinterpret_cast<int*>(s_stats + kStatFloats);
  const uint32_t s_bar = smem_u32(s_flag + 4);   // kStages mbarriers: the pre-split B half of each stage has landed

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int n0 = blockIdx.x * BN, m0 = blockIdx.y * BM;
  const int k_begin = blockIdx.z * a.k_per_slice;
  const int k_end = min(a.K, k_begin + a.k_per_slice);
  const int n_kb = (k_end - k_begin + BK - 1) / BK;

  Pos pa[4], pb[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    pa[j] = pos_of(a.a_mn, warp, lane, j);
    pb[j] = pos_of(a.b_mn, warp, lane, j);
  }
  // kPrefetch k-blocks of global loads stay in flight per thread (register ring) so the HBM/L2 latency is paid
  // once per tile, not once per k-block.
  float4 va[kPf][4], vb[kPreB ? 1 : kPf][4];
  auto issue = [&](int kb, float4 (&xa)[4], float4 (&xb)[4]) {
    const int k0 = k_begin + kb * BK;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      xa[j] = load_pos(a.A, a.lda, a.a_mn, pa[j], m0, a.M, k0, k_end);
      // B rows past the MMA width are never read by the tensor core
      if constexpr (!kPreB)
        xb[j] = pb[j].mn < NM ? load_pos(a.B, a.ldb, a.b_mn, pb[j], n0, a.N, k0, k_end)
                              : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto stage_out = [&](int kb, const float4 (&xa)[4], const float4 (&xb)[4]) {
    const int k0 = k_begin + kb * BK;
    const uint32_t st = smem_base + (uint32_t)(kb % kStages) * kStageBytes;
    store_block(st, a.a_mn, pa, xa, BM, m0, a.M, k0, k_end);
    if constexpr (!kPreB) store_block(st + 2 * kTileBytes, a.b_mn, pb, xb, NM, n0, a.N, k0, k_end);
  };
  // pre-split B: k-block kb's two planes -> stage kb % kStages (thread 0; the stage's previous wgmma's have retired)
  auto issue_b = [&](int kb) {
    constexpr uint32_t kPlaneBytes = NM * BK * 4;
    const uint32_t st = smem_base + (uint32_t)(kb % kStages) * kStageBytes + 2 * kTileBytes;
    const uint32_t bar = s_bar + 8u * (uint32_t)(kb % kStages);
    const long long off = (long long)blockIdx.x * a.b_tile_floats + (long long)(k_begin / BK + kb) * (NM * BK);
    mbar_expect_tx(bar, 2 * kPlaneBytes);
    bulk_g2s(st, a.b_hi + off, kPlaneBytes, bar);
    bulk_g2s(st + kTileBytes, a.b_lo + off, kPlaneBytes, bar);
  };
  if constexpr (kPreB) {
    if (tid == 0) {
      for (int s = 0; s < kStages; ++s) mbar_init(s_bar + 8u * s, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
  }

  float acc[R], acc2[R];
#pragma unroll
  for (int i = 0; i < R; ++i) acc[i] = acc2[i] = 0.f;

  er_pdl_wait();
  if (kPreB && tid == 0 && n_kb > 0) issue_b(0);
#pragma unroll
  for (int u = 0; u < kPf; ++u)
    if (u < n_kb) issue(u, va[u], vb[kPreB ? 0 : u]);

  for (int kb0 = 0; kb0 < n_kb; kb0 += kPf) {
#pragma unroll
    for (int u = 0; u < kPf; ++u) {
      const int kb = kb0 + u;
      if (kb < n_kb) {
        stage_out(kb, va[u], vb[kPreB ? 0 : u]);
        if (kb + kPf < n_kb) issue(kb + kPf, va[u], vb[kPreB ? 0 : u]);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> tensor core
        __syncthreads();
        if constexpr (kPreB) {
          // past this barrier both warpgroups have retired the wgmma's of k-block kb - 2: its stage takes kb + 1
          if (tid == 0 && kb + 1 < n_kb) issue_b(kb + 1);
          mbar_wait(s_bar + 8u * (uint32_t)(kb % kStages), (uint32_t)(kb / kStages) & 1u);
        }
        const uint32_t st = smem_base + (uint32_t)(kb % kStages) * kStageBytes;
        const uint32_t a_hi = st + (uint32_t)wg * (64u * 128u), b_hi = st + 2 * kTileBytes;
        fence_regs(acc);
        fence_regs(acc2);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < BK / 8; ++kk) {
          const uint64_t ahi = make_desc(a_hi + kk * 32), alo = make_desc(a_hi + kTileBytes + kk * 32);
          const uint64_t bhi = make_desc(b_hi + kk * 32), blo = make_desc(b_hi + kTileBytes + kk * 32);
          wgmma_tf32(acc2, alo, bhi);
          wgmma_tf32(acc2, ahi, blo);
          wgmma_tf32(acc, ahi, bhi);
        }
        wgmma_commit();
        wgmma_wait<1>();
        fence_regs(acc);
        fence_regs(acc2);
      }
    }
  }
  wgmma_wait<0>();
  fence_regs(acc);
  fence_regs(acc2);
  __syncthreads();   // both warpgroups are done with the stage ring: it becomes the output tile

  // ===== epilogue: registers -> shared tile [128][kOutPitch] -> global =====
  float* tile = reinterpret_cast<float*>(base_ptr);
  {
    // accumulator fragment: register i of warp w (of the warpgroup) holds row 16w + lane/4 + 8*((i/2)%2),
    // column 8*(i/4) + 2*(lane%4) + i%2
    const int rbase = 64 * wg + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
    for (int i = 0; i < R; i += 2) {
      const int row = rbase + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * (lane & 3);
      *reinterpret_cast<float2*>(tile + row * kOutPitch + col) = make_float2(acc[i] + acc2[i], acc[i + 1] + acc2[i + 1]);
    }
  }
  __syncthreads();
  float* out = a.n_slices > 1 ? a.partials + (long long)blockIdx.z * a.M * a.N : a.C;
  const long long ldo = a.n_slices > 1 ? (long long)a.N : a.ldc;
  const bool vec_ok = (ldo & 3) == 0 && ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
  const int m_tiles = gridDim.y;
  const int n_live = min(NM, a.N - n0);
  // ---- batch-norm statistics: publish this tile's partials and take a ticket BEFORE the big stores, so the
  // fence only has to cover 1.5 KB of partials ----
  if (a.bn_part) {
    // thread = (column tid % 128, row half tid / 128): one pass of shifted sums (shift = the half's first value,
    // so no E[x^2]-E[x]^2 cancellation), then the two halves merge in order
    const int cl = tid & 127, half = tid >> 7;
    const int nv = min(64, a.M - (m0 + 64 * half));   // valid rows of this half (<= 0: none)
    if (cl < n_live) {
      const float* tc = tile + (64 * half) * kOutPitch + cl;
      const float shift = nv > 0 ? tc[0] : 0.f;
      float sd0 = 0.f, sd1 = 0.f, sq0 = 0.f, sq1 = 0.f;
#pragma unroll 8
      for (int rr = 0; rr < 64; rr += 2) {
        const float v0 = tc[rr * kOutPitch] - shift, v1 = tc[(rr + 1) * kOutPitch] - shift;
        if (rr < nv) { sd0 += v0; sq0 += v0 * v0; }
        if (rr + 1 < nv) { sd1 += v1; sq1 += v1 * v1; }
      }
      const float fn = (float)max(nv, 1);
      const float sd = sd0 + sd1;
      float* sst = s_stats + (half * 128 + cl) * 3;
      sst[0] = (float)max(nv, 0);
      sst[1] = shift + sd / fn;
      sst[2] = fmaxf((sq0 + sq1) - sd * sd / fn, 0.f);
    }
    __syncthreads();
    if (tid < n_live) {
      Welford t = {s_stats[tid * 3], s_stats[tid * 3 + 1], s_stats[tid * 3 + 2]};
      const float* p = s_stats + (128 + tid) * 3;
      wf_merge(t, Welford{p[0], p[1], p[2]});
      float* gp = a.bn_part + ((long long)blockIdx.y * a.N + n0 + tid) * 3;
      __stcg(gp, t.n); __stcg(gp + 1, t.mean); __stcg(gp + 2, t.m2);
      __threadfence();
    }
    __syncthreads();
    if (tid == 0) *s_flag = (atomicAdd(a.bn_counter + blockIdx.x, 1u) == (unsigned)(m_tiles - 1));
  }
  // ---- shared -> global: a warp stores NM/4 16 B units of a row, rows in turn ----
  {
    const bool add_bias = a.bias != nullptr && a.n_slices == 1;
    constexpr int kUnits = NM / 4;
#pragma unroll 4
    for (int i = tid; i < BM * kUnits; i += kThreads) {
      const int rr = i / kUnits, u = i % kUnits;
      const int grow = m0 + rr, col = n0 + 4 * u;
      if (grow >= a.M || col >= a.N) continue;
      float4 v = *reinterpret_cast<const float4*>(tile + rr * kOutPitch + 4 * u);
      if (add_bias) {
        v.x += a.bias[col];
        if (col + 1 < a.N) v.y += a.bias[col + 1];
        if (col + 2 < a.N) v.z += a.bias[col + 2];
        if (col + 3 < a.N) v.w += a.bias[col + 3];
      }
      float* orow = out + (long long)grow * ldo;
      if (vec_ok && col + 3 < a.N) {
        *reinterpret_cast<float4*>(orow + col) = v;
      } else {
        orow[col] = v.x;
        if (col + 1 < a.N) orow[col + 1] = v.y;
        if (col + 2 < a.N) orow[col + 2] = v.z;
        if (col + 3 < a.N) orow[col + 3] = v.w;
      }
    }
  }
  if (a.bn_part) {
    __syncthreads();
    if (*s_flag) {
      // Last row-tile of this column tile: combine the per-tile (n, mean, M2) of its columns.  Two threads per
      // column (even / odd tiles), two passes (global mean, then M2 about it) whose loads are independent - the
      // whole merge costs a few L2 round trips instead of one per tile - fixed order.
      __threadfence();
      const int cl2 = tid & 127, half = tid >> 7;
      const int col = n0 + cl2;
      const bool live = cl2 < n_live;
      float* s_red = s_stats;                           // reuse: [2][128] floats per pass
      float cnt = 0.f, wsum = 0.f;
      if (live) {
#pragma unroll 16
        for (int mt = half; mt < m_tiles; mt += 2) {
          const float* gp = a.bn_part + ((long long)mt * a.N + col) * 3;
          const float n = __ldcg(gp), mu = __ldcg(gp + 1);
          cnt += n;
          wsum += n * mu;
        }
      }
      s_red[half * 128 + cl2] = cnt;
      s_red[256 + half * 128 + cl2] = wsum;
      __syncthreads();
      const float n_tot = s_red[cl2] + s_red[128 + cl2];
      const float mean_z = (s_red[256 + cl2] + s_red[384 + cl2]) / fmaxf(n_tot, 1.f);
      float m2 = 0.f;
      if (live) {
#pragma unroll 16
        for (int mt = half; mt < m_tiles; mt += 2) {
          const float* gp = a.bn_part + ((long long)mt * a.N + col) * 3;
          const float n = __ldcg(gp), mu = __ldcg(gp + 1), q2 = __ldcg(gp + 2);
          const float d = mu - mean_z;
          m2 += q2 + n * d * d;
        }
      }
      s_red[512 + half * 128 + cl2] = m2;
      __syncthreads();
      if (live && half == 0) {
        const float mean = mean_z + (a.bn.bias ? a.bn.bias[col] : 0.f);
        const float var = (s_red[512 + cl2] + s_red[640 + cl2]) / n_tot;   // biased (tf.layers.batch_normalization)
        a.bn.save_mean[col] = mean;
        a.bn.save_rstd[col] = 1.0f / sqrtf(var + a.bn.eps);
        if (a.bn.moving_mean) {
          a.bn.moving_mean[col] = a.bn.moving_mean[col] * a.bn.momentum + mean * (1.f - a.bn.momentum);
          a.bn.moving_var[col] = a.bn.moving_var[col] * a.bn.momentum + var * (1.f - a.bn.momentum);
        }
      }
      if (tid == 0) a.bn_counter[blockIdx.x] = 0u;
    }
  }
}

// C[m,n] = sum_s partials[s][m][n] (+ bias[n]), fixed order.
__global__ void splitk_reduce_kernel(const float* __restrict__ partials, const float* __restrict__ bias,
                                     float* __restrict__ C, long long ldc, int M, int N, int n_slices) {
  er_pdl_wait();
  const long long total = (long long)M * N;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int m = (int)(i / N), n = (int)(i % N);
    float acc = partials[i];
    for (int s = 1; s < n_slices; ++s) acc += partials[(long long)s * total + i];
    if (bias) acc += bias[n];
    C[(long long)m * ldc + n] = acc;
  }
}

// Split K when the output has too few tiles to occupy the SMs (the dW GEMMs: K = batch).
static void plan(int64_t M, int64_t N, int64_t K, int* n_slices, int* k_per_slice) {
  const int64_t tiles = ceil_div(M, BM) * ceil_div(N, BN);
  const int64_t kblocks = ceil_div(K, BK);
  int64_t s = 1;
  if (tiles * 2 <= kSmCount && kblocks >= 16) {
    s = kSmCount / tiles;
    s = std::min<int64_t>(s, kblocks / 8);   // at least 8 k-blocks (256 k) per slice
    s = std::max<int64_t>(s, 1);
  }
  const int64_t per = ceil_div(kblocks, s);
  *k_per_slice = (int)(per * BK);
  *n_slices = (int)ceil_div(kblocks, per);
}

template <int NM, bool kPreB>
static int launch(const Args& a, dim3 grid, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_tf32x3_kernel<NM, kPreB>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kSmemBytes);
    if (e != cudaSuccess) return er::fail(ER_ERR_CUDA, std::string("er_gemm: ") + cudaGetErrorString(e));
    attr_set = true;
  }
  er::launch_pdl(gemm_tf32x3_kernel<NM, kPreB>, grid, dim3(kThreads), (size_t)kSmemBytes, st, a);
  return ER_OK;
}
template <bool kPreB>
static int launch_width(const Args& a, dim3 grid, cudaStream_t st) {
  switch (mma_width(a.N)) {
    case 128: return launch<128, kPreB>(a, grid, st);
    case 64: return launch<64, kPreB>(a, grid, st);
    case 32: return launch<32, kPreB>(a, grid, st);
    default: return launch<16, kPreB>(a, grid, st);
  }
}

// One thread per 16 B chunk of a plane pair: chunk c of row r of k-block kb holds the 4 k's of swizzle slot
// c ^ (r % 8); elements past the operand's rows / K are zeros (what mask_chunk gives the in-kernel split).
constexpr int kMaxPlaneJobs = 32;
struct PlaneJobs {
  er_gemm_plane_t j[kMaxPlaneJobs];
};
__global__ void split_planes_kernel(PlaneJobs jobs) {
  const er_gemm_plane_t p = jobs.j[blockIdx.y];
  const int nm = mma_width(p.rows);
  const long long n_kb = (p.k + BK - 1) / BK;
  const long long chunks = (p.rows + BN - 1) / BN * n_kb * nm * (BK / 4);
  er_pdl_wait();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < chunks; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i & 7);
    const long long rk = i >> 3;                  // (tile, kb, r) row of 32 k
    const int r = (int)(rk % nm);
    const long long tkb = rk / nm;
    const long long row = tkb / n_kb * nm + r, k0 = tkb % n_kb * BK + 4 * (c ^ (r & 7));
    float v[4], hi[4], lo[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      v[e] = row < p.rows && k0 + e < p.k ? p.src[row * p.ld_row + (k0 + e) * p.ld_k] : 0.f;
      split_tf32(v[e], hi[e], lo[e]);
    }
    reinterpret_cast<float4*>(p.hi)[i] = make_float4(hi[0], hi[1], hi[2], hi[3]);
    reinterpret_cast<float4*>(p.lo)[i] = make_float4(lo[0], lo[1], lo[2], lo[3]);
  }
}

}  // namespace gemm
}  // namespace er

extern "C" size_t er_gemm_workspace_bytes(int64_t M, int64_t N, int64_t K) {
  int s, kp;
  er::gemm::plan(M, N, K, &s, &kp);
  return s > 1 ? (size_t)s * (size_t)M * (size_t)N * sizeof(float) : 0;
}

extern "C" size_t er_gemm_bn_workspace_bytes(int64_t M, int64_t N);

// B is given either in memory (B, ldb, b_mn_major) or as pre-split planes (b_hi, b_lo; B NULL)
static int gemm_impl(const float* A, int64_t lda, int32_t a_mn_major, const float* B, int64_t ldb,
                     int32_t b_mn_major, const float* b_hi, const float* b_lo, const float* bias, float* C,
                     int64_t ldc, int64_t M, int64_t N, int64_t K, const er_bn_stats_t* bn, void* ws,
                     size_t ws_bytes, er_stream_t stream) {
  using namespace er::gemm;
  const bool pre_b = B == nullptr;
  ER_REQUIRE(A && C && (pre_b ? b_hi && b_lo : true), "null operand");
  ER_REQUIRE(M > 0 && N > 0 && K > 0 && M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31), "bad shape");
  ER_REQUIRE((lda & 3) == 0 && (pre_b || (ldb & 3) == 0), "operand pitch must be a multiple of 4 floats");
  ER_REQUIRE((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(b_hi) & 15) == 0 && (reinterpret_cast<uintptr_t>(b_lo) & 15) == 0,
             "operands must be 16-byte aligned");
  // a pitch shorter than the row would read the next row's first elements as this row's last ones
  ER_REQUIRE(lda >= (a_mn_major ? M : K) && (pre_b || ldb >= (b_mn_major ? N : K)), "pitch smaller than row");
  ER_REQUIRE(ldc >= N, "ldc < N");
  Args a;
  a.A = A; a.B = B; a.C = C; a.bias = bias;
  a.b_hi = b_hi; a.b_lo = b_lo; a.b_tile_floats = plane_tile_floats(N, K);
  a.lda = lda; a.ldb = ldb; a.ldc = ldc;
  a.M = (int)M; a.N = (int)N; a.K = (int)K;
  a.a_mn = a_mn_major ? 1 : 0; a.b_mn = b_mn_major ? 1 : 0;
  plan(M, N, K, &a.n_slices, &a.k_per_slice);
  a.partials = nullptr;
  a.bn_part = nullptr;
  a.bn_counter = nullptr;
  if (a.n_slices > 1) {
    ER_REQUIRE(!bn, "batch-norm statistics need an unsplit K (er_gemm_workspace_bytes(M,N,K) == 0)");
    ER_REQUIRE(ws && ws_bytes >= er_gemm_workspace_bytes(M, N, K), "workspace too small");
    a.partials = static_cast<float*>(ws);
  }
  if (bn) {
    ER_REQUIRE(bn->save_mean && bn->save_rstd, "bn: save_mean / save_rstd missing");
    ER_REQUIRE((bn->moving_mean == nullptr) == (bn->moving_var == nullptr), "bn: moving_mean and moving_var go together");
    ER_REQUIRE(ws && ws_bytes >= er_gemm_bn_workspace_bytes(M, N), "bn workspace too small");
    a.bn = *bn;
    a.bn_counter = static_cast<unsigned int*>(ws);
    a.bn_part = reinterpret_cast<float*>(static_cast<char*>(ws) + 1024);
  }
  cudaStream_t st = er::as_stream(stream);
  dim3 grid((unsigned)er::ceil_div(N, BN), (unsigned)er::ceil_div(M, BM), (unsigned)a.n_slices);
  const int rc = pre_b ? launch_width<true>(a, grid, st) : launch_width<false>(a, grid, st);
  if (rc != ER_OK) return rc;
  int launches = 1;
  if (a.n_slices > 1) {
    const long long total = (long long)M * N;
    int blocks = (int)std::min<long long>((total + 255) / 256, 4LL * er::kSmCount);
    er::launch_pdl(splitk_reduce_kernel, dim3(blocks), dim3(256), 0, st, (const float*)a.partials, bias, C,
                   (long long)ldc, (int)M, (int)N, a.n_slices);
    ++launches;
  }
  er::count_launches(launches);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_gemm(const float* A, int64_t lda, int32_t a_mn_major, const float* B, int64_t ldb,
                       int32_t b_mn_major, const float* bias, float* C, int64_t ldc, int64_t M, int64_t N,
                       int64_t K, void* ws, size_t ws_bytes, er_stream_t stream) {
  ER_REQUIRE(B, "null operand");
  return gemm_impl(A, lda, a_mn_major, B, ldb, b_mn_major, nullptr, nullptr, bias, C, ldc, M, N, K, nullptr, ws,
                   ws_bytes, stream);
}

extern "C" size_t er_gemm_bn_workspace_bytes(int64_t M, int64_t N) {
  return 1024 + (size_t)er::ceil_div(M, er::gemm::BM) * (size_t)N * 3 * sizeof(float);
}

extern "C" int er_gemm_bn(const float* A, int64_t lda, int32_t a_mn_major, const float* B, int64_t ldb,
                          int32_t b_mn_major, float* C, int64_t ldc, int64_t M, int64_t N, int64_t K,
                          const er_bn_stats_t* bn, void* ws, size_t ws_bytes, er_stream_t stream) {
  if (!bn) return er::fail(ER_ERR_INVALID_ARG, "er_gemm_bn: bn is NULL");
  if (er::ceil_div(N, er::gemm::BN) > 256) return er::fail(ER_ERR_INVALID_ARG, "er_gemm_bn: N too large");
  ER_REQUIRE(B, "null operand");
  return gemm_impl(A, lda, a_mn_major, B, ldb, b_mn_major, nullptr, nullptr, nullptr, C, ldc, M, N, K, bn, ws,
                   ws_bytes, stream);
}

extern "C" size_t er_gemm_plane_floats(int64_t rows, int64_t K) {
  if (rows <= 0 || K <= 0) return 0;
  return (size_t)er::ceil_div(rows, (int64_t)er::gemm::BN) * (size_t)er::gemm::plane_tile_floats(rows, K);
}

extern "C" int er_gemm_split_planes(const er_gemm_plane_t* planes, int32_t n, er_stream_t stream) {
  using namespace er::gemm;
  ER_REQUIRE(n >= 0 && (n == 0 || planes), "bad plane list");
  cudaStream_t st = er::as_stream(stream);
  int launches = 0;
  for (int i0 = 0; i0 < n; i0 += kMaxPlaneJobs) {
    PlaneJobs jobs;
    const int cnt = std::min(kMaxPlaneJobs, n - i0);
    long long max_chunks = 0;
    for (int i = 0; i < cnt; ++i) {
      const er_gemm_plane_t& p = planes[i0 + i];
      ER_REQUIRE(p.src && p.hi && p.lo, "null plane pointer");
      ER_REQUIRE(p.rows > 0 && p.k > 0 && p.rows < (1ll << 31) && p.k < (1ll << 31), "bad plane shape");
      ER_REQUIRE((reinterpret_cast<uintptr_t>(p.hi) & 15) == 0 && (reinterpret_cast<uintptr_t>(p.lo) & 15) == 0,
                 "planes must be 16-byte aligned");
      jobs.j[i] = p;
      max_chunks = std::max<long long>(max_chunks, (long long)er_gemm_plane_floats(p.rows, p.k) / 4);
    }
    const int blocks = (int)std::min<long long>((max_chunks + 255) / 256, 2LL * er::kSmCount);
    er::launch_pdl(split_planes_kernel, dim3(blocks, cnt), dim3(256), 0, st, jobs);
    ++launches;
  }
  er::count_launches(launches);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

extern "C" int er_gemm_planes(const float* A, int64_t lda, int32_t a_mn_major, const float* b_hi, const float* b_lo,
                              const float* bias, float* C, int64_t ldc, int64_t M, int64_t N, int64_t K,
                              const er_bn_stats_t* bn, void* ws, size_t ws_bytes, er_stream_t stream) {
  if (bn && bias) return er::fail(ER_ERR_INVALID_ARG, "er_gemm_planes: with bn the bias goes in bn->bias");
  if (bn && er::ceil_div(N, er::gemm::BN) > 256) return er::fail(ER_ERR_INVALID_ARG, "er_gemm_planes: N too large");
  return gemm_impl(A, lda, a_mn_major, nullptr, 0, 0, b_hi, b_lo, bias, C, ldc, M, N, K, bn, ws, ws_bytes, stream);
}
