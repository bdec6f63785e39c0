// points.cu -- nearest-neighbour search of the point-transfer path (sm_90a), SURVEY.md 8(f) rank 4.
//
// reference: models/spatial_transformers/spatial_transformer.py:655-668 (`congeal_points`, flow STN): for every key point
// the nearest sampling-grid entry is found by brute force -- the reference materialises the (N, H, W, P) distance tensor
//     dist = |p|^2 + |g|^2 - 2 g.p          (the EXPANDED form, :663-666)
// and takes `argmin` over the H*W grid entries (first minimum wins), then `unravel_index`.  At P ~ 4e5 points (config 4) that
// tensor is 26 GB per sample.  Here nothing is materialised: a CTA holds a tile of grid entries (gx, gy, |g|^2) in shared
// memory, every thread owns one point and scans the tile keeping (distance, index) with a strict `<` (first minimum), and
// the pixel range is split across CTAs whose results meet in ONE 64-bit atomicMin per point on the packed key
// (order-preserving bits of the distance << 32 | index): smaller distance wins, equal distances resolve to the smaller
// index -- exactly argmin's rule.  The distance is evaluated with the reference's expanded expression and operation order
// (separately rounded products, no FMA contraction), so near-ties resolve like the reference's.
#include "common.cuh"
#include "points.cuh"

namespace gg {
namespace {

constexpr int kNNThreads = 256;
constexpr int kNNTile = 1024;     // grid entries per shared-memory tile

__device__ __forceinline__ unsigned order_bits(float f) {   // monotone map float -> unsigned (handles negative rounding noise)
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__global__ void nn_init_kernel(unsigned long long* __restrict__ best, int64_t total) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < total) best[i] = ~0ull;
}

__global__ void __launch_bounds__(kNNThreads)
nn_argmin_kernel(unsigned long long* __restrict__ best, const float* __restrict__ grid, const float* __restrict__ points,
                 int64_t P, int HW, int splits) {
  __shared__ float sgx[kNNTile], sgy[kNNTile], sgg[kNNTile];
  const int64_t n = blockIdx.z;
  const int split = blockIdx.y;
  const int64_t pt = static_cast<int64_t>(blockIdx.x) * kNNThreads + threadIdx.x;
  const int per = (HW + splits - 1) / splits;
  const int e0 = split * per, e1 = min(e0 + per, HW);
  float px = 0.f, py = 0.f, pp = 0.f;
  if (pt < P) {
    px = __ldg(points + (n * P + pt) * 2);
    py = __ldg(points + (n * P + pt) * 2 + 1);
    pp = __fadd_rn(__fmul_rn(px, px), __fmul_rn(py, py));          // pts.pow(2).sum(-1)
  }
  float bd = INFINITY;
  int bi = 0x7fffffff;
  const float* g = grid + n * HW * 2;
  for (int t0 = e0; t0 < e1; t0 += kNNTile) {
    const int cnt = min(kNNTile, e1 - t0);
    __syncthreads();
    for (int i = threadIdx.x; i < cnt; i += kNNThreads) {
      const float2 v = __ldg(reinterpret_cast<const float2*>(g + static_cast<int64_t>(t0 + i) * 2));
      sgx[i] = v.x; sgy[i] = v.y;
      sgg[i] = __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y));   // g.pow(2).sum(-1)
    }
    __syncthreads();
    if (pt < P) {
#pragma unroll 4
      for (int i = 0; i < cnt; ++i) {
        const float sim = __fadd_rn(__fmul_rn(sgx[i], px), __fmul_rn(sgy[i], py));      // (g @ p)
        const float d = __fsub_rn(__fadd_rn(pp, sgg[i]), __fmul_rn(2.f, sim));         // |p|^2 + |g|^2 - 2 sim
        if (d < bd) { bd = d; bi = t0 + i; }
      }
    }
  }
  if (pt < P && bi != 0x7fffffff) {
    const unsigned long long key = (static_cast<unsigned long long>(order_bits(bd)) << 32) | static_cast<unsigned>(bi);
    atomicMin(best + n * P + pt, key);
  }
}

__global__ void nn_unpack_kernel(int64_t* __restrict__ index, const unsigned long long* __restrict__ best, int64_t total) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < total) index[i] = static_cast<int64_t>(best[i] & 0xffffffffull);
}

}  // namespace

int nn_argmin_search(unsigned long long* best, const float* grid, const float* points, int64_t N, int64_t P, int HW,
                     cudaStream_t st) {
  const int64_t total = N * P;
  nn_init_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(best, total);
  GG_CHECK_LAUNCH("nn_init launch");
  const int64_t pblocks = (P + kNNThreads - 1) / kNNThreads;
  if (pblocks > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "nn_argmin: too many points");
  // split the grid entries over CTAs until the machine is filled ~2x (each split scans >= one tile)
  int splits = static_cast<int>((2LL * sm_count() + pblocks * N - 1) / (pblocks * N));
  const int max_splits = (HW + kNNTile - 1) / kNNTile;
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  if (splits > 65535) splits = 65535;
  nn_argmin_kernel<<<dim3(static_cast<unsigned>(pblocks), static_cast<unsigned>(splits), static_cast<unsigned>(N)), kNNThreads, 0, st>>>(
      best, grid, points, P, HW, splits);
  GG_CHECK_LAUNCH("nn_argmin launch");
  return GG_OK;
}

}  // namespace gg

using namespace gg;

extern "C" {

int64_t gg_nn_argmin_workspace(int64_t N, int64_t P) { return (N > 0 && P > 0) ? N * P * 8 : 0; }

int gg_nn_argmin(int64_t* index, void* workspace, const float* grid, const float* points, int64_t N, int64_t P, int HW,
                 void* stream) {
  if (N < 0 || P < 0 || HW < 0) return fail(GG_ERR_BAD_ARG, "nn_argmin: negative size");
  if (N * P == 0) return GG_OK;
  if (HW == 0) return fail(GG_ERR_BAD_ARG, "nn_argmin: empty grid (argmin of an empty set)");
  if (!index || !workspace || !grid || !points) return fail(GG_ERR_BAD_ARG, "nn_argmin: null tensor");
  if (N > 65535) return fail(GG_ERR_UNSUPPORTED, "nn_argmin: batch > 65535");
  auto st = static_cast<cudaStream_t>(stream);
  auto* best = static_cast<unsigned long long*>(workspace);
  const int64_t total = N * P;
  const int rc = nn_argmin_search(best, grid, points, N, P, HW, st);
  if (rc != GG_OK) return rc;
  nn_unpack_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(index, best, total);
  GG_CHECK_LAUNCH("nn_unpack launch");
  return GG_OK;
}

}  // extern "C"
