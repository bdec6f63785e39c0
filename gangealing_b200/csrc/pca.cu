// pca.cu -- per-block fp64 column means and centred Gram matrices of an fp32 row matrix (sm_90a).
//
//   gg_batch_gram   for each row block [off[b], off[b+1]) of a row-major (n, D) fp32 matrix W:
//                     mean[b]  = fp64 column mean of the block
//                     gram[b]  = sum over the block's rows of (x - mean[b]) (x - mean[b])^T, the full symmetric D x D matrix
//                   These are the per-batch terms of the Gram form of sklearn's IncrementalPCA (training/latent_learner.py):
//                   they do not depend on the running fit, so every batch of a 10^6-row fit is one launch here and only
//                   the chain of D x D eigensolves that consumes them stays sequential.
//
// Two kernels:
//   1. means: one CTA per (64-column strip, block); four row groups sum rows r, r+4, ... in fp64, then the four partial
//      sums are added in a fixed order.  No atomics: bitwise reproducible.
//   2. Gram:  one CTA per (upper-triangle 64 x 64 tile, block), 4 warps of 32 x 32.  fp32 rows are staged in shared memory
//      with cp.async, converted to fp64 with the block mean subtracted (rows past the block's end become zeros), and the
//      tile is accumulated with the fp64 tensor-core MMA (mma.sync m16n8k16 .f64, SASS DMMA) over the block's rows in
//      order.  Each off-diagonal tile is written twice, at (i, j) and mirrored at (j, i).  No atomics: bitwise
//      reproducible.
#include "common.cuh"

namespace gg {
namespace {

constexpr int kTile = 64;           // output tile edge (columns of W per operand)
constexpr int kRows = 32;           // rows of W per pipeline stage (two k16 MMA steps)
constexpr int kPad = 8;             // fp64 row padding: row stride 72 doubles keeps fragment loads bank-conflict free
constexpr int kStride = kTile + kPad;
constexpr int kGramThreads = 128;
constexpr int kMeanThreads = 256;
constexpr int kBlocksPerLaunch = 256;   // row-block offsets travel in the kernel's parameters (257 x 8 bytes)
constexpr int kMaxD = 1024;

struct Blocks {
  int64_t off[kBlocksPerLaunch + 1];
};

// byte size of the Gram kernel's dynamic shared memory
constexpr int kStageFloats = kRows * 2 * kTile;                 // fp32 staging: both operands' 64 columns of 32 rows
constexpr int kSmemBytes = kStageFloats * 4 + 2 * kRows * kStride * 8 + 2 * kTile * 8;

__global__ void __launch_bounds__(kMeanThreads)
block_mean_kernel(double* __restrict__ mean, const float* __restrict__ w, Blocks blocks, int D) {
  __shared__ double part[kMeanThreads];
  const int b = blockIdx.y;
  const int col = blockIdx.x * kTile + (threadIdx.x & (kTile - 1));
  const int grp = threadIdx.x / kTile;
  const int64_t r0 = blocks.off[b], r1 = blocks.off[b + 1];
  double s = 0.0;
  for (int64_t r = r0 + grp; r < r1; r += kMeanThreads / kTile) s += static_cast<double>(w[r * D + col]);
  part[threadIdx.x] = s;
  __syncthreads();
  if (grp == 0) {
    double t = part[threadIdx.x];
#pragma unroll
    for (int g = 1; g < kMeanThreads / kTile; ++g) t += part[threadIdx.x + g * kTile];
    mean[static_cast<int64_t>(b) * D + col] = t / static_cast<double>(r1 - r0);
  }
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// D(16x8) += A(16x16) B(16x8), fp64.  Fragments (g = lane / 4, t = lane % 4):
//   a[i] = A[g + 8 (i % 2)][t + 4 (i / 2)],  b[i] = B[t + 4 i][g],  d[i] = D[g + 8 (i / 2)][2 t + i % 2]
__device__ __forceinline__ void dmma16816(double (&d)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
      "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
      : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}

// the (ti, tj), ti <= tj, tile of linear index `lin` in row-major order of the upper triangle of a T x T tile grid
__device__ __forceinline__ void upper_tile(int lin, int T, int& ti, int& tj) {
  ti = 0;
  while (lin >= T - ti) { lin -= T - ti; ++ti; }
  tj = ti + lin;
}

__global__ void __launch_bounds__(kGramThreads)
block_gram_kernel(double* __restrict__ gram, const double* __restrict__ mean, const float* __restrict__ w, Blocks blocks,
                  int D) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* stage = reinterpret_cast<float*>(smem_raw);                         // [kRows][2 * kTile] fp32
  double* xa = reinterpret_cast<double*>(stage + kStageFloats);              // [kRows][kStride] centred fp64, columns ti
  double* xb = xa + kRows * kStride;                                         // [kRows][kStride] centred fp64, columns tj
  double* mu = xb + kRows * kStride;                                         // [2 * kTile] the two strips' means

  const int T = D / kTile;
  int ti, tj;
  upper_tile(blockIdx.x, T, ti, tj);
  const bool diag = ti == tj;
  const int b = blockIdx.y;
  const int64_t r0 = blocks.off[b], r1 = blocks.off[b + 1];
  const int tid = threadIdx.x;
  const int ca = ti * kTile, cb = tj * kTile;
  const double* mean_b = mean + static_cast<int64_t>(b) * D;
  mu[tid] = mean_b[(tid < kTile ? ca : cb - kTile) + tid];

  // staging: 32 rows x (64 + 64) fp32 = 1024 16-byte chunks, 8 per thread; chunk q: row q / 32, 16-byte column q % 32
  // (columns 0-15 of the chunk row belong to strip ti, 16-31 to strip tj; the diagonal tile stages strip ti only)
  auto issue = [&](int64_t row0) {
#pragma unroll
    for (int k = 0; k < kRows * 2 * kTile / 4 / kGramThreads; ++k) {
      const int q = tid + k * kGramThreads;
      const int r = q >> 5, c4 = q & 31;
      const int64_t row = row0 + r;
      if (row < r1 && (!diag || c4 < 16)) {
        const int col = c4 < 16 ? ca + 4 * c4 : cb + 4 * (c4 - 16);
        cp_async16(stage + r * 2 * kTile + 4 * c4, w + row * D + col);
      }
    }
    cp_async_commit();
  };

  const int lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
  double acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.0;

  const double* xbs = diag ? xa : xb;
  issue(r0);
  for (int64_t row0 = r0; row0 < r1; row0 += kRows) {
    cp_async_wait_all();
    __syncthreads();                 // stage holds rows [row0, row0 + 32); every warp is done with the previous fp64 tiles
    // convert + centre: element e = tid + k * 128 of the 32 x 128 stage (zeros past the block's end)
#pragma unroll 4
    for (int k = 0; k < kRows * 2 * kTile / kGramThreads; ++k) {
      const int e = tid + k * kGramThreads;
      const int r = e >> 7, c = e & 127;
      if (diag && c >= kTile) continue;
      const double v = row0 + r < r1 ? static_cast<double>(stage[e]) - mu[c] : 0.0;
      (c < kTile ? xa : xb)[r * kStride + (c & (kTile - 1))] = v;
    }
    __syncthreads();                 // fp64 tiles complete; the stage is free for the next rows
    if (row0 + kRows < r1) issue(row0 + kRows);
#pragma unroll
    for (int k0 = 0; k0 < kRows; k0 += 16) {
      double af[2][8], bf[4][4];
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int q = 0; q < 8; ++q) af[i][q] = xa[(k0 + t + 4 * (q >> 1)) * kStride + wm + 16 * i + g + 8 * (q & 1)];
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q) bf[j][q] = xbs[(k0 + t + 4 * q) * kStride + wn + 8 * j + g];
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) dmma16816(acc[i][j], af[i], bf[j]);
    }
  }

  double* out = gram + static_cast<int64_t>(b) * D * D;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int m = ca + wm + 16 * i + g + 8 * (e >> 1);
        const int n = cb + wn + 8 * j + 2 * t + (e & 1);
        out[static_cast<int64_t>(m) * D + n] = acc[i][j][e];
        if (!diag) out[static_cast<int64_t>(n) * D + m] = acc[i][j][e];
      }
}

}  // namespace
}  // namespace gg

using namespace gg;

extern "C" GG_API int gg_batch_gram(double* gram, double* mean, const float* w, const int64_t* batch_offsets, int64_t B,
                                    int D, void* stream) {
  if (!gram || !mean || !w || !batch_offsets) return fail(GG_ERR_BAD_ARG, "gg_batch_gram: null pointer");
  if (B <= 0 || D <= 0) return fail(GG_ERR_BAD_ARG, "gg_batch_gram: B = %lld and D = %d must be positive",
                                    static_cast<long long>(B), D);
  if (D % kTile != 0 || D > kMaxD)
    return fail(GG_ERR_UNSUPPORTED, "gg_batch_gram: D = %d must be a multiple of %d and at most %d", D, kTile, kMaxD);
  if (reinterpret_cast<uintptr_t>(w) % 16 != 0) return fail(GG_ERR_BAD_ARG, "gg_batch_gram: w is not 16-byte aligned");
  if (batch_offsets[0] < 0) return fail(GG_ERR_BAD_ARG, "gg_batch_gram: offsets[0] = %lld is negative",
                                        static_cast<long long>(batch_offsets[0]));
  for (int64_t b = 0; b < B; ++b)
    if (batch_offsets[b + 1] <= batch_offsets[b])
      return fail(GG_ERR_BAD_ARG, "gg_batch_gram: offsets must increase (offsets[%lld] = %lld, offsets[%lld] = %lld)",
                  static_cast<long long>(b), static_cast<long long>(batch_offsets[b]), static_cast<long long>(b + 1),
                  static_cast<long long>(batch_offsets[b + 1]));
  static DeviceOnce once;
  if (once.needed()) {
    const cudaError_t e = cudaFuncSetAttribute(block_gram_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
    if (e != cudaSuccess) return cuda_fail(e, "gg_batch_gram: cudaFuncSetAttribute");
    once.done();
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int T = D / kTile;
  for (int64_t b0 = 0; b0 < B; b0 += kBlocksPerLaunch) {
    const int nb = static_cast<int>(B - b0 < kBlocksPerLaunch ? B - b0 : kBlocksPerLaunch);
    Blocks blocks;
    for (int i = 0; i <= nb; ++i) blocks.off[i] = batch_offsets[b0 + i];
    block_mean_kernel<<<dim3(T, nb), kMeanThreads, 0, st>>>(mean + b0 * D, w, blocks, D);
    GG_CHECK_LAUNCH("gg_batch_gram: mean kernel");
    block_gram_kernel<<<dim3(T * (T + 1) / 2, nb), kGramThreads, kSmemBytes, st>>>(gram + b0 * D * D, mean + b0 * D, w,
                                                                                  blocks, D);
    GG_CHECK_LAUNCH("gg_batch_gram: Gram kernel");
  }
  return 0;
}
