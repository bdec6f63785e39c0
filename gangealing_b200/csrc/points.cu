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
// Non-finite distances follow torch.argmin too: a NaN counts as smaller than any number and the first NaN wins (every NaN
// packs to the smallest key, 0 in the high word, so the splits merge by index alone), and a point whose distances are all
// +inf resolves to index 0 (each split starts from its first entry, so every point issues its atomicMin).
#include "common.cuh"
#include "points.cuh"

namespace gg {
namespace {

constexpr int kNNThreads = 256;
constexpr int kNNTile = 1024;     // grid entries per shared-memory tile

__device__ __forceinline__ unsigned order_bits(float f) {   // monotone map float -> unsigned (handles negative rounding noise)
  if (f != f) return 0u;                                    // every NaN below -inf's key (0x007fffff): argmin's rule
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// argmin's order: `d` replaces the best `bd` so far if it is smaller, or if it is the first NaN
__device__ __forceinline__ bool argmin_better(float d, float bd) { return d < bd || (d != d && bd == bd); }

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
  float bd = INFINITY;   // with bi = e0: the split's first entry, unless an entry is smaller or NaN
  int bi = e0;
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
        if (argmin_better(d, bd)) { bd = d; bi = t0 + i; }
      }
    }
  }
  if (pt < P && e0 < e1) {
    const unsigned long long key = (static_cast<unsigned long long>(order_bits(bd)) << 32) | static_cast<unsigned>(bi);
    atomicMin(best + n * P + pt, key);
  }
}

__global__ void nn_unpack_kernel(int64_t* __restrict__ index, const unsigned long long* __restrict__ best, int64_t total) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < total) index[i] = static_cast<int64_t>(best[i] & 0xffffffffull);
}

// ---------------------------------------------------------------- windowed point tracking over lerped grids
// vis_correspondence.py:59-114 (`pad_grid`, `nearest_neighbor_within_patch`) once per frame of smoothly_sample_image
// (:183-205), for all T frames of a stage in one launch: one thread per point, its patch centre carried in registers.
// Frame t's grid is lerp(base, target, alphas[t]) (torch.lerp's formula, as warp.cu MODE 3), seen through pad_grid's
// (H+2) x (W+2) linear-extrapolation ring; window positions beyond the ring are Unfold's zero padding, (0, 0) candidates.
// The window's argmin follows torch.argmin as the search above does: the first NaN wins, an all-+inf window picks its first
// candidate.
__device__ __forceinline__ float lerp_aten(float a, float b, float w) {
  const float d = b - a;
  return (fabsf(w) < 0.5f) ? fmaf(w, d, a) : fmaf(-d, 1.f - w, b);
}

// Value of pad_grid(lerp(base, target, w)) at padded position (qy, qx), 0 <= qy < H+2, 0 <= qx < W+2.  The ring holds
// 2 g[1] - g[2] style extrapolations of the replicate-padded grid; the column pass is assigned last, so it owns the corners.
__device__ __forceinline__ float2 padded_at(const float* __restrict__ base, const float* __restrict__ target, int H, int W,
                                            float w, int qy, int qx) {
  auto g = [&](int y, int x) {
    const int64_t i = (static_cast<int64_t>(y) * W + x) * 2;
    const float2 a = __ldg(reinterpret_cast<const float2*>(base + i));
    const float2 b = __ldg(reinterpret_cast<const float2*>(target + i));
    return make_float2(lerp_aten(a.x, b.x, w), lerp_aten(a.y, b.y, w));
  };
  auto extrap = [](float2 a, float2 b) {   // 2 a - b, each op rounded as torch does it
    return make_float2(__fsub_rn(__fmul_rn(2.f, a.x), b.x), __fsub_rn(__fmul_rn(2.f, a.y), b.y));
  };
  const int y = min(max(qy - 1, 0), H - 1);
  if (qx == 0) return extrap(g(y, 0), g(y, 1));
  if (qx == W + 1) return extrap(g(y, W - 1), g(y, W - 2));
  const int x = qx - 1;
  if (qy == 0) return extrap(g(0, x), g(1, x));
  if (qy == H + 1) return extrap(g(H - 1, x), g(H - 2, x));
  return g(qy - 1, x);
}

__device__ __forceinline__ int64_t floor_mod(int64_t a, int64_t m) {
  const int64_t r = a % m;
  return r < 0 ? r + m : r;
}

__device__ __forceinline__ int64_t floor_div(int64_t a, int64_t m) {
  return (a - floor_mod(a, m)) / m;
}

__global__ void __launch_bounds__(128)
track_points_kernel(int64_t* __restrict__ track, int64_t* __restrict__ centers, const float* __restrict__ base,
                    const float* __restrict__ target, const float* __restrict__ alphas, const float* __restrict__ points,
                    int T, int64_t N, int64_t P, int H, int W, int patch) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= N * P) return;
  const int64_t n = i / P;
  const float* bn = base + n * H * static_cast<int64_t>(W) * 2;
  const float* tn = target + n * H * static_cast<int64_t>(W) * 2;
  const float px = __ldg(points + i * 2), py = __ldg(points + i * 2 + 1);
  const float pp = __fadd_rn(__fmul_rn(px, px), __fmul_rn(py, py));       // points.pow(2).sum(-1)
  const int hp = H + 2, wp = W + 2, r = patch / 2;
  int64_t cx = centers[i * 2], cy = centers[i * 2 + 1];
  for (int t = 0; t < T; ++t) {
    const float w = __ldg(alphas + t);
    // flat index of the padded centre with grid.size(1) = H + 2 as the row stride; Unfold's patch of that index sits at
    // (row, col) = divmod(flat, W + 2)
    const int64_t flat = (cx + 1) + hp * (cy + 1);
    const int64_t ly = flat / wp, lx = flat - ly * wp;
    float bd = INFINITY;
    int bk = 0;
    for (int ky = 0; ky < patch; ++ky) {
      const int64_t qy = ly + ky - r;
      for (int kx = 0; kx < patch; ++kx) {
        const int64_t qx = lx + kx - r;
        float2 g = make_float2(0.f, 0.f);   // Unfold's zero padding
        if (qy >= 0 && qy < hp && qx >= 0 && qx < wp) g = padded_at(bn, tn, H, W, w, static_cast<int>(qy), static_cast<int>(qx));
        const float sim = __fadd_rn(__fmul_rn(g.x, px), __fmul_rn(g.y, py));
        const float gg = __fadd_rn(__fmul_rn(g.x, g.x), __fmul_rn(g.y, g.y));
        const float d = __fsub_rn(__fadd_rn(pp, gg), __fmul_rn(2.f, sim));
        if (argmin_better(d, bd)) { bd = d; bk = ky * patch + kx; }   // bk = 0 seeds the first candidate
      }
    }
    // unravel over (patch, patch) -> (kx, ky); offset (kx - r) + (H + 2)(ky - r); unravel over (H + 2, W + 2) (floor
    // division: a window leaving the padded grid wraps), minus the padding
    const int64_t out = flat + (bk % patch - r) + static_cast<int64_t>(hp) * (bk / patch - r);
    cx = floor_mod(out, wp) - 1;
    cy = floor_mod(floor_div(out, wp), hp) - 1;
    int64_t* tr = track + ((static_cast<int64_t>(t) * N * P) + i) * 2;
    tr[0] = cx;
    tr[1] = cy;
  }
  centers[i * 2] = cx;
  centers[i * 2 + 1] = cy;
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

int gg_track_points_lerp(int64_t* track, int64_t* centers, const float* base, const float* target, const float* alphas,
                         const float* points, int T, int64_t N, int64_t P, int H, int W, int patch, void* stream) {
  if (N < 0 || P < 0) return fail(GG_ERR_BAD_ARG, "track_points_lerp: negative size");
  if (T < 1) return fail(GG_ERR_BAD_ARG, "track_points_lerp: T (frames) must be >= 1, got %d", T);
  if (H != W) return fail(GG_ERR_BAD_ARG, "track_points_lerp: the grid must be square (H == W), got %d x %d", H, W);
  if (H < 2) return fail(GG_ERR_BAD_ARG, "track_points_lerp: the grid must be at least 2 x 2");
  if (patch < 1 || patch % 2 == 0) return fail(GG_ERR_BAD_ARG, "track_points_lerp: patch must be odd and >= 1, got %d", patch);
  if (!track || !centers || !base || !target || !alphas || !points) return fail(GG_ERR_BAD_ARG, "track_points_lerp: null tensor");
  const int64_t total = N * P;
  if (total == 0) return GG_OK;
  if ((total + 127) / 128 > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "track_points_lerp: too many points");
  track_points_kernel<<<static_cast<unsigned>((total + 127) / 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      track, centers, base, target, alphas, points, T, N, P, H, W, patch);
  GG_CHECK_LAUNCH("track_points launch");
  return GG_OK;
}

}  // extern "C"
