// splat.cu -- Gaussian forward splatting of points into an image (sm_90a).
//
// Replaces reference utils/splat2d_cuda/src/splat_gpu_impl.cu:41-96 (one 32-thread block per 32 points,
// (C+1) scalar float atomics per footprint pixel) and the five ATen passes of splat_gpu.c:20-41
// (zeros, clone, clamp, add, divide).
//
//  * accumulators are interleaved per pixel -- slot 0 = sum of alpha, slots 1..C = sum of alpha*value[c],
//    padded to a multiple of 4 floats -- so one footprint pixel receives ONE 16-byte vector reduction
//    (red.global.add.v4.f32, sm_90+) per group of 4 slots instead of C+1 scalar atomics: a quarter of the reference's
//    atomic traffic for RGB colours (C = 3) or a mask (C = 1);
//  * one thread per point, 64-thread CTAs (a dense mask of 4e5 points fills the machine, a sparse one of 2.5e4 still
//    spreads over ~400 CTAs), fire-and-forget reductions: no return value, no ordering between them;
//  * normalisation (input + sum) / (alpha [clamped >= 1 if soft] + 1e-8) and the NCHW re-layout are one fused pass.
// Cross-point aggregation was built twice and measured slower BOTH times, so it is not here:
//   - round 1: one lane per point, same-pixel lanes merged per footprint step with match.any + a segmented shuffle scan --
//     0.55-0.75x the reference at sigma 1.3 (r02_opbench_vs_reference_b32_before.txt): the merge cost more than it saved;
//   - round 2a: a "torus" of per-lane register accumulators walking raster-ordered points (one flush per pixel when the
//     footprint window moves off it) -- 0.72-0.85x the reference in 3 of 4 config-4 cases (r02_opbench_vs_reference_b32.json):
//     all 32 lanes execute bookkeeping for every point while a sigma-0.3 footprint has 9 pixels;
//   - round 2b (this kernel): 1.3-1.7x the reference in all four cases (r02_splat_modes.txt).  At the dense end (4e5 points,
//     7x7 footprints: 19.8 M vector reductions in 81 us = 244 G/s) the scatter runs at the L2's reduction rate; the v4 form
//     is what moved the needle, not merging.
// Float atomics make the summation order (hence the last bits) run-to-run dependent, exactly as in the
// reference; the SET of touched pixels is deterministic.
// HBM: algorithmic bytes 4*N*(P*(2+C) + (C+1)*H*W + 2*C*H*W); the scatter itself is L2-reduction-bound.
#include <algorithm>

#include "common.cuh"
#include "grid.cuh"
#include "lookup.cuh"

namespace gg {
namespace {

struct SplatParams {
  int64_t n;
  int64_t points;   // P
  int c, h, w;
  int slots;        // (C + 1) rounded up to a multiple of 4
};

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// One thread per point, one 16-byte reduction per footprint pixel and group of 4 accumulator slots (GROUPS = 1: C <= 3,
// GROUPS = 2: C <= 7).  Same footprint schedule as the reference kernel (splat_gpu_impl.cu:60-94: rows t..b, columns l..r).
template <int GROUPS, bool LOOKUP>
__global__ void __launch_bounds__(64)
splat_direct_kernel(float* __restrict__ acc, const float* __restrict__ coords, const float* __restrict__ values,
                    const float* __restrict__ sigma, SplatParams p, int64_t total, LookupParams lk) {
  const int64_t index = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (index >= total) return;
  const int64_t n = index / p.points;
  float2 xy = __ldg(reinterpret_cast<const float2*>(coords + index * 2));
  if (LOOKUP) {
    xy = lookup_point(lk, n, xy.x, xy.y);
    if (lk.points_out) *reinterpret_cast<float2*>(lk.points_out + index * 2) = xy;
  }
  const float x = xy.x, y = xy.y;
  // points outside the image are ignored (splat_gpu_impl.cu:76); bounds: :78-81
  if (!(x >= 0.f && x < static_cast<float>(p.w) && y >= 0.f && y < static_cast<float>(p.h))) return;
  const float sd = __ldg(sigma + n), len = 2.f * sd, norm = -1.f / (2.f * sd * sd);
  const int t = static_cast<int>(fmaxf(0.f, floorf(y - len))), b = static_cast<int>(fminf(static_cast<float>(p.h - 1), ceilf(y + len)));
  const int l = static_cast<int>(fmaxf(0.f, floorf(x - len))), r = static_cast<int>(fminf(static_cast<float>(p.w - 1), ceilf(x + len)));
  const float* val = values + index * p.c;
  float v[GROUPS * 4];
  v[0] = 1.f;                                             // slot 0 accumulates alpha itself
#pragma unroll
  for (int q = 1; q < GROUPS * 4; ++q) v[q] = (q <= p.c) ? __ldg(val + q - 1) : 0.f;
  float* acc_n = acc + n * p.h * static_cast<int64_t>(p.w) * (GROUPS * 4);
  for (int py = t; py <= b; ++py) {
    const float ddy = static_cast<float>(py) - y;
    float* row = acc_n + static_cast<int64_t>(py) * p.w * (GROUPS * 4);
    for (int px = l; px <= r; ++px) {
      const float ddx = static_cast<float>(px) - x;
      const float a = expf(norm * (ddx * ddx + ddy * ddy));
      float* dst = row + px * (GROUPS * 4);
#pragma unroll
      for (int g = 0; g < GROUPS; ++g) red_add_v4(dst + 4 * g, a * v[4 * g], a * v[4 * g + 1], a * v[4 * g + 2], a * v[4 * g + 3]);
    }
  }
}

// generic channel count: scalar atomics per slot (C > 7); still interleaved accumulators
__global__ void __launch_bounds__(256)
splat_scatter_generic_kernel(float* __restrict__ acc, const float* __restrict__ coords, const float* __restrict__ values,
                             const float* __restrict__ sigma, SplatParams p, int64_t total) {
  for (int64_t index = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; index < total;
       index += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t n = index / p.points;
    const float x = coords[index * 2], y = coords[index * 2 + 1];
    if (!(x >= 0.f && x < static_cast<float>(p.w) && y >= 0.f && y < static_cast<float>(p.h))) continue;
    const float sd = sigma[n], len = 2.f * sd, norm = -1.f / (2.f * sd * sd);
    const int t = static_cast<int>(fmaxf(0.f, floorf(y - len)));
    const int b = static_cast<int>(fminf(static_cast<float>(p.h - 1), ceilf(y + len)));
    const int l = static_cast<int>(fmaxf(0.f, floorf(x - len)));
    const int r = static_cast<int>(fminf(static_cast<float>(p.w - 1), ceilf(x + len)));
    const float* val = values + index * p.c;
    float* acc_n = acc + n * p.h * static_cast<int64_t>(p.w) * p.slots;
    for (int py = t; py <= b; ++py)
      for (int px = l; px <= r; ++px) {
        const float ddx = static_cast<float>(px) - x, ddy = static_cast<float>(py) - y;
        const float alpha = expf(norm * (ddx * ddx + ddy * ddy));
        float* dst = acc_n + (static_cast<int64_t>(py) * p.w + px) * p.slots;
        atomicAdd(dst, alpha);
        for (int c = 0; c < p.c; ++c) atomicAdd(dst + 1 + c, alpha * val[c]);
      }
  }
}

// out[n,c,y,x] = (input[n,c,y,x] + acc[n,y,x,1+c]) / (alpha' + 1e-8)     (splat_gpu.c:36-41)
__global__ void __launch_bounds__(256)
splat_normalize_kernel(float* __restrict__ out, const float* __restrict__ input, const float* __restrict__ acc,
                       SplatParams p, int soft, int64_t total) {
  for (int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t hw = static_cast<int64_t>(p.h) * p.w;
    const int64_t pix = idx % hw;
    const int64_t nc = idx / hw;
    const int c = static_cast<int>(nc % p.c);
    const int64_t n = nc / p.c;
    const float* a = acc + (n * hw + pix) * p.slots;
    float alpha = a[0];
    if (soft) alpha = fmaxf(alpha, 1.f);
    out[idx] = (input[idx] + a[1 + c]) / (alpha + 1e-8f);
  }
}

// ---------------------------------------------------------------------------------------------------- composited grids
// The label-propagation animation (reference vis_correspondence.py:133-158): for every (frame, image) the two splats of
// splat_points (helpers.py:178-187, colours and soft-normalised alpha), the alpha composite, then images2grid
// (helpers.py:39-43: make_grid(normalize=True, range=(-1, 1)) and the uint8 quantisation), in one scatter launch and one
// composite launch per chunk of frames.  Both splats weigh a footprint pixel with the same Gaussian a, so one pass
// accumulates [sum a, sum a*r, sum a*g, sum a*b] and, with an alpha channel, [sum a*alpha, 0, 0, 0]: one or two 16-byte
// reductions per footprint pixel.  Without an alpha channel sum a*alpha = sum a and the second group is not allocated.
struct GridParams {
  int64_t n, points;          // N images per frame, P points per image
  int r;                      // image side
  GridLayout g;               // make_grid layout of one frame (grid.cuh)
  int colors_n, alpha_n;      // 1 (broadcast) or N
  float sigma, opacity;
};

// LOOKUP (gg_splat_lookup_composite_grid, one frame): the points arrive as query coordinates in the congealed frame,
// (query_n in {1, N}, P, 2), and are looked up in image n's sampling grid (lookup.cuh), then mirrored where flip[n] is set
// (reference applications/propagate_to_images.py:64-69: uncongeal_points on the flipped image, x -> (R - 1) - x).
struct FrameLookup {
  LookupParams lk;
  const unsigned char* flip;  // (N,) or null
  int query_n;                // 1 (broadcast) or N
};

// One thread per (frame, image, point); the footprint schedule and bounds test of splat_direct_kernel.
template <bool ALPHA, bool LOOKUP>
__global__ void __launch_bounds__(64)
splat_frames_kernel(float* __restrict__ acc, const float* __restrict__ coords, const float* __restrict__ colors,
                    const float* __restrict__ alpha, GridParams p, int64_t total, FrameLookup fl) {
  constexpr int SLOTS = ALPHA ? 8 : 4;
  const int64_t index = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (index >= total) return;
  const int64_t image = index / p.points;            // (frame, image) within the chunk
  const int64_t pt = index - image * p.points;
  const int64_t n = image % p.n;
  float2 xy;
  if (LOOKUP) {
    const float2 q = __ldg(reinterpret_cast<const float2*>(coords + ((fl.query_n == 1 ? 0 : n) * p.points + pt) * 2));
    xy = lookup_point(fl.lk, n, q.x, q.y);
    if (fl.flip && fl.flip[n]) xy.x = static_cast<float>(p.r - 1) - xy.x;
    if (fl.lk.points_out) *reinterpret_cast<float2*>(fl.lk.points_out + index * 2) = xy;
  } else {
    xy = __ldg(reinterpret_cast<const float2*>(coords + index * 2));
  }
  const float x = xy.x, y = xy.y;
  const int h = p.r, w = p.r;
  if (!(x >= 0.f && x < static_cast<float>(w) && y >= 0.f && y < static_cast<float>(h))) return;
  const float sd = p.sigma, len = 2.f * sd, norm = -1.f / (2.f * sd * sd);
  const int t = static_cast<int>(fmaxf(0.f, floorf(y - len))), b = static_cast<int>(fminf(static_cast<float>(h - 1), ceilf(y + len)));
  const int l = static_cast<int>(fmaxf(0.f, floorf(x - len))), r = static_cast<int>(fminf(static_cast<float>(w - 1), ceilf(x + len)));
  const float* col = colors + ((p.colors_n == 1 ? 0 : n) * p.points + pt) * 3;
  const float cr = __ldg(col), cg = __ldg(col + 1), cb = __ldg(col + 2);
  const float al = ALPHA ? __ldg(alpha + (p.alpha_n == 1 ? 0 : n) * p.points + pt) : 0.f;
  float* acc_n = acc + image * h * static_cast<int64_t>(w) * SLOTS;
  for (int py = t; py <= b; ++py) {
    const float ddy = static_cast<float>(py) - y;
    float* row = acc_n + static_cast<int64_t>(py) * w * SLOTS;
    for (int px = l; px <= r; ++px) {
      const float ddx = static_cast<float>(px) - x;
      const float a = expf(norm * (ddx * ddx + ddy * ddy));
      float* dst = row + px * SLOTS;
      red_add_v4(dst, a * 1.f, a * cr, a * cg, a * cb);
      if (ALPHA) red_add_v4(dst + 4, a * al, 0.f, 0.f, 0.f);
    }
  }
}

// One output pixel (3 bytes, HWC) of one frame's grid per thread.  SPLAT: composite the accumulated splats over the image
// as splat2d's normalisation and splat_points' blend do, every operation rounded on its own:
//   obj = S_c / (A + 1e-8);  m = (S_alpha / (max(A, 1) + 1e-8)) * opacity;  v = m * obj + (1 - m) * img.
template <bool SPLAT, bool ALPHA>
__global__ void __launch_bounds__(256)
composite_grid_kernel(unsigned char* __restrict__ out, const float* __restrict__ acc, const float* __restrict__ images,
                      GridParams p, int64_t total) {
  constexpr int SLOTS = ALPHA ? 8 : 4;
  const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int gx = static_cast<int>(idx % p.g.wg);
  const int64_t rest = idx / p.g.wg;
  const int gy = static_cast<int>(rest % p.g.hg);
  const int64_t frame = rest / p.g.hg;
  unsigned char* o = out + idx * 3;
  int y, x;
  const int64_t k = grid_source(p.g, gx, gy, y, x);
  if (k < 0) {   // make_grid's padding (pad value 0)
    o[0] = o[1] = o[2] = 0;
    return;
  }
  const int64_t image = frame * p.n + k;
  const int64_t plane = static_cast<int64_t>(p.r) * p.r, pix = static_cast<int64_t>(y) * p.r + x;
  const float* img = images + image * 3 * plane + pix;
  float v[3] = {__ldg(img), __ldg(img + plane), __ldg(img + 2 * plane)};
  if (SPLAT) {
    const float* a = acc + (image * plane + pix) * SLOTS;
    const float4 s = __ldg(reinterpret_cast<const float4*>(a));
    const float sa = ALPHA ? __ldg(a + 4) : s.x;
    const float den = __fadd_rn(s.x, 1e-8f);
    const float m = __fmul_rn(__fdiv_rn(sa, __fadd_rn(fmaxf(s.x, 1.f), 1e-8f)), p.opacity);
    const float keep = __fsub_rn(1.f, m);
    const float sc[3] = {s.y, s.z, s.w};
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = __fadd_rn(__fmul_rn(m, __fdiv_rn(sc[c], den)), __fmul_rn(keep, v[c]));
  }
  o[0] = quantise_range(v[0], -1.f, 1.f);   // images2grid: make_grid(normalize=True, range=(-1, 1))
  o[1] = quantise_range(v[1], -1.f, 1.f);
  o[2] = quantise_range(v[2], -1.f, 1.f);
}

inline int splat_grid(int64_t total, int threads) {
  int64_t g = (total + threads - 1) / threads;
  const int64_t cap = static_cast<int64_t>(sm_count()) * 8;
  return static_cast<int>(g < cap ? (g > 0 ? g : 1) : cap);
}

}  // namespace
}  // namespace gg

using namespace gg;

extern "C" {

int64_t gg_splat2d_workspace(int64_t N, int C, int H, int W) {
  if (N < 0 || C < 0 || H < 0 || W < 0) return -1;
  const int slots = ((C + 1) + 3) / 4 * 4;
  return N * H * static_cast<int64_t>(W) * slots * static_cast<int64_t>(sizeof(float));
}

static int splat_impl(float* out, void* workspace, const float* input, const float* coordinates, const float* values,
                      const float* sigma, int64_t N, int64_t P, int C, int H, int W, int soft_normalize, const LookupParams* lk,
                      void* stream) {
  if (N < 0 || P < 0 || C < 0 || H < 0 || W < 0) return fail(GG_ERR_BAD_ARG, "splat2d: negative size");
  const int64_t numel = N * C * H * static_cast<int64_t>(W);
  if (numel == 0) return GG_OK;  // reference returns the (empty) clone (splat_gpu.c:23-26)
  if (!out || !input || !workspace || !sigma) return fail(GG_ERR_BAD_ARG, "splat2d: null tensor");
  if (P > 0 && (!coordinates || !values)) return fail(GG_ERR_BAD_ARG, "splat2d: null points");
  auto st = static_cast<cudaStream_t>(stream);
  SplatParams p;
  p.n = N; p.points = P; p.c = C; p.h = H; p.w = W;
  p.slots = ((C + 1) + 3) / 4 * 4;
  if (lk && p.slots != 4)
    return fail(GG_ERR_UNSUPPORTED, "splat2d_lookup: the fused lookup serves C <= 3 (the call sites splat RGB colours or a 1-channel mask)");
  // only the direct kernel performs the lookup, and it addresses the accumulators with 32-bit pixel offsets
  if (lk && static_cast<int64_t>(H) * W * p.slots >= 0x7fffffffLL)
    return fail(GG_ERR_UNSUPPORTED, "splat2d_lookup: H * W * 4 accumulator slots must stay below 2^31 (the fused lookup's scatter)");
  cudaError_t e = cudaMemsetAsync(workspace, 0, static_cast<size_t>(gg_splat2d_workspace(N, C, H, W)), st);
  if (e != cudaSuccess) return cuda_fail(e, "splat2d workspace memset");
  float* acc = static_cast<float*>(workspace);
  const int64_t total = N * P;
  if (total > 0) {
    if (p.slots <= 8 && static_cast<int64_t>(H) * W * p.slots < 0x7fffffffLL) {
      const int64_t blocks = (total + 63) / 64;
      if (blocks > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "splat2d: too many points");
      const unsigned g = static_cast<unsigned>(blocks);
      if (lk) splat_direct_kernel<1, true><<<g, 64, 0, st>>>(acc, coordinates, values, sigma, p, total, *lk);
      else if (p.slots == 4) splat_direct_kernel<1, false><<<g, 64, 0, st>>>(acc, coordinates, values, sigma, p, total, LookupParams{});
      else splat_direct_kernel<2, false><<<g, 64, 0, st>>>(acc, coordinates, values, sigma, p, total, LookupParams{});
    } else {
      splat_scatter_generic_kernel<<<splat_grid(total, 256), 256, 0, st>>>(acc, coordinates, values, sigma, p, total);
    }
    GG_CHECK_LAUNCH("splat_scatter launch");
  }
  splat_normalize_kernel<<<splat_grid(numel, 256), 256, 0, st>>>(out, input, acc, p, soft_normalize ? 1 : 0, numel);
  GG_CHECK_LAUNCH("splat_normalize launch");
  return GG_OK;
}

int gg_splat2d_forward(float* out, void* workspace, const float* input, const float* coordinates, const float* values,
                       const float* sigma, int64_t N, int64_t P, int C, int H, int W, int soft_normalize,
                       void* stream) {
  return splat_impl(out, workspace, input, coordinates, values, sigma, N, P, C, H, W, soft_normalize, nullptr, stream);
}

int gg_splat2d_lookup_forward(float* out, float* points_out, void* workspace, const float* input, const float* grid,
                              const float* query, const float* values, const float* sigma, int64_t N, int64_t P, int C,
                              int H, int W, int grid_h, int grid_w, float unnorm_k, float unnorm_m, int soft_normalize,
                              void* stream) {
  if (grid_h < 1 || grid_w < 1 || !(unnorm_k != 0.f)) return fail(GG_ERR_BAD_ARG, "splat2d_lookup: bad grid geometry");
  if (N * P > 0 && !grid) return fail(GG_ERR_BAD_ARG, "splat2d_lookup: null grid");
  LookupParams lk;
  lk.grid = grid; lk.gh = grid_h; lk.gw = grid_w; lk.k = unnorm_k; lk.m = unnorm_m; lk.points_out = points_out;
  return splat_impl(out, workspace, input, query, values, sigma, N, P, C, H, W, soft_normalize, &lk, stream);
}

int64_t gg_splat_composite_grid_workspace(int64_t T_chunk, int64_t N, int R, int has_alpha) {
  if (T_chunk < 0 || N < 0 || R < 0) return -1;
  return T_chunk * N * R * static_cast<int64_t>(R) * (has_alpha ? 8 : 4) * static_cast<int64_t>(sizeof(float));
}

int gg_splat_composite_grid(unsigned char* out, void* workspace, int64_t workspace_bytes, const float* images,
                            const float* points, const float* colors, const float* alpha, float sigma, float opacity,
                            int64_t T, int64_t N, int64_t P, int C, int R, int nrow, int padding, int colors_n, int alpha_n,
                            void* stream) {
  constexpr int64_t kIntMax = 0x7fffffffLL;
  if (T < 0 || N < 1 || P < 0 || R < 1 || nrow < 1 || padding < 0)
    return fail(GG_ERR_BAD_ARG, "splat_composite_grid: T, P, padding >= 0 and N, R, nrow >= 1");
  if (C != 3) return fail(GG_ERR_BAD_ARG, "splat_composite_grid: C must be 3 (RGB images and colours)");
  if (!(sigma > 0.f)) return fail(GG_ERR_BAD_ARG, "splat_composite_grid: sigma must be > 0");
  if (!(opacity >= 0.f && opacity <= 1.f)) return fail(GG_ERR_BAD_ARG, "splat_composite_grid: opacity must lie in [0, 1]");
  if (T > 0 && (!out || !images)) return fail(GG_ERR_BAD_ARG, "splat_composite_grid: null output or images");
  const bool splat = P > 0 && T > 0;
  const bool has_alpha = alpha != nullptr;
  if (splat && (!points || !colors || !workspace)) return fail(GG_ERR_BAD_ARG, "splat_composite_grid: null points, colors or workspace");
  if (splat && (colors_n != 1 && colors_n != N)) return fail(GG_ERR_BAD_ARG, "splat_composite_grid: colors_n must be 1 or N");
  if (splat && has_alpha && (alpha_n != 1 && alpha_n != N)) return fail(GG_ERR_BAD_ARG, "splat_composite_grid: alpha_n must be 1 or N");
  if (splat && (reinterpret_cast<uintptr_t>(workspace) % 16 != 0))
    return fail(GG_ERR_BAD_ARG, "splat_composite_grid: workspace must be 16-byte aligned (vector reductions)");
  if (splat && (reinterpret_cast<uintptr_t>(points) % 8 != 0))
    return fail(GG_ERR_BAD_ARG, "splat_composite_grid: points must be 8-byte aligned");
  GridParams p;
  p.n = N; p.points = P; p.r = R;
  const int slots = has_alpha ? 8 : 4;
  const int64_t frame_acc = N * R * static_cast<int64_t>(R) * slots;
  if (!make_grid_layout(p.g, N, R, R, nrow, padding) || frame_acc > kIntMax || N * 3 * R * static_cast<int64_t>(R) > kIntMax ||
      N * P > kIntMax)
    return fail(GG_ERR_BAD_ARG, "splat_composite_grid: one frame's grid, images, accumulators or points exceed 2^31 elements");
  const int64_t hg = p.g.hg, wg = p.g.wg;
  p.colors_n = colors_n; p.alpha_n = alpha_n; p.sigma = sigma; p.opacity = opacity;
  const int64_t frame_bytes = frame_acc * static_cast<int64_t>(sizeof(float));
  // frames per launch: as many as the workspace holds, with every launch's thread count below 2^31
  int64_t chunk = std::min(T, kIntMax / std::max(splat ? N * P : 1, hg * wg));
  if (splat) {
    if (workspace_bytes < frame_bytes)
      return fail(GG_ERR_BAD_ARG, "splat_composite_grid: the workspace holds less than one frame's accumulators");
    chunk = std::min(chunk, workspace_bytes / frame_bytes);
  }
  if (T == 0) return GG_OK;
  auto st = static_cast<cudaStream_t>(stream);
  float* acc = static_cast<float*>(workspace);
  for (int64_t t0 = 0; t0 < T; t0 += chunk) {
    const int64_t tc = T - t0 < chunk ? T - t0 : chunk;
    const int64_t pix = tc * hg * wg;
    const float* img = images + t0 * N * 3 * R * static_cast<int64_t>(R);
    unsigned char* o = out + t0 * hg * wg * 3;
    const unsigned blocks = static_cast<unsigned>((pix + 255) / 256);
    if (splat) {
      cudaError_t e = cudaMemsetAsync(acc, 0, static_cast<size_t>(tc * frame_bytes), st);
      if (e != cudaSuccess) return cuda_fail(e, "splat_composite_grid workspace memset");
      const int64_t total = tc * N * P;
      const unsigned sblocks = static_cast<unsigned>((total + 63) / 64);
      const float* pts = points + t0 * N * P * 2;
      if (has_alpha) {
        splat_frames_kernel<true, false><<<sblocks, 64, 0, st>>>(acc, pts, colors, alpha, p, total, FrameLookup{});
        GG_CHECK_LAUNCH("splat_frames launch");
        composite_grid_kernel<true, true><<<blocks, 256, 0, st>>>(o, acc, img, p, pix);
      } else {
        splat_frames_kernel<false, false><<<sblocks, 64, 0, st>>>(acc, pts, colors, nullptr, p, total, FrameLookup{});
        GG_CHECK_LAUNCH("splat_frames launch");
        composite_grid_kernel<true, false><<<blocks, 256, 0, st>>>(o, acc, img, p, pix);
      }
    } else {
      composite_grid_kernel<false, false><<<blocks, 256, 0, st>>>(o, nullptr, img, p, pix);
    }
    GG_CHECK_LAUNCH("composite_grid launch");
  }
  return GG_OK;
}

int gg_splat_lookup_composite_grid(unsigned char* out, float* points_out, void* workspace, int64_t workspace_bytes,
                                   const float* images, const float* grid, const float* query, const unsigned char* flip,
                                   const float* colors, const float* alpha, float sigma, float opacity, int64_t N, int64_t P,
                                   int query_n, int C, int R, int grid_h, int grid_w, int nrow, int padding, int colors_n,
                                   int alpha_n, void* stream) {
  constexpr int64_t kIntMax = 0x7fffffffLL;
  if (N < 1 || P < 0 || R < 1 || nrow < 1 || padding < 0 || grid_h < 1 || grid_w < 1)
    return fail(GG_ERR_BAD_ARG, "splat_lookup_composite_grid: P, padding >= 0 and N, R, nrow, grid_h, grid_w >= 1");
  if (C != 3) return fail(GG_ERR_BAD_ARG, "splat_lookup_composite_grid: C must be 3 (RGB images and colours)");
  if (!(sigma > 0.f)) return fail(GG_ERR_BAD_ARG, "splat_lookup_composite_grid: sigma must be > 0");
  if (!(opacity >= 0.f && opacity <= 1.f))
    return fail(GG_ERR_BAD_ARG, "splat_lookup_composite_grid: opacity must lie in [0, 1]");
  if (!out || !images) return fail(GG_ERR_BAD_ARG, "splat_lookup_composite_grid: null output or images");
  const bool splat = P > 0;
  const bool has_alpha = alpha != nullptr;
  if (splat && (!grid || !query || !colors || !workspace))
    return fail(GG_ERR_BAD_ARG, "splat_lookup_composite_grid: null grid, query, colors or workspace");
  if (splat && query_n != 1 && query_n != N) return fail(GG_ERR_BAD_ARG, "splat_lookup_composite_grid: query_n must be 1 or N");
  if (splat && colors_n != 1 && colors_n != N) return fail(GG_ERR_BAD_ARG, "splat_lookup_composite_grid: colors_n must be 1 or N");
  if (splat && has_alpha && alpha_n != 1 && alpha_n != N)
    return fail(GG_ERR_BAD_ARG, "splat_lookup_composite_grid: alpha_n must be 1 or N");
  if (splat && reinterpret_cast<uintptr_t>(workspace) % 16 != 0)
    return fail(GG_ERR_BAD_ARG, "splat_lookup_composite_grid: workspace must be 16-byte aligned (vector reductions)");
  if (splat && (reinterpret_cast<uintptr_t>(query) % 8 != 0 || reinterpret_cast<uintptr_t>(grid) % 8 != 0 ||
                reinterpret_cast<uintptr_t>(points_out) % 8 != 0))
    return fail(GG_ERR_BAD_ARG, "splat_lookup_composite_grid: query, grid and points_out must be 8-byte aligned");
  GridParams p;
  p.n = N; p.points = P; p.r = R;
  const int slots = has_alpha ? 8 : 4;
  const int64_t frame_acc = N * R * static_cast<int64_t>(R) * slots;
  if (!make_grid_layout(p.g, N, R, R, nrow, padding) || frame_acc > kIntMax || N * 3 * R * static_cast<int64_t>(R) > kIntMax ||
      N * P > kIntMax)
    return fail(GG_ERR_BAD_ARG, "splat_lookup_composite_grid: the grid, images, accumulators or points exceed 2^31 elements");
  const int64_t frame_bytes = frame_acc * static_cast<int64_t>(sizeof(float));
  if (splat && workspace_bytes < frame_bytes)
    return fail(GG_ERR_BAD_ARG, "splat_lookup_composite_grid: the workspace holds less than the grid's accumulators");
  p.colors_n = colors_n; p.alpha_n = alpha_n; p.sigma = sigma; p.opacity = opacity;
  FrameLookup fl;
  // uncongeal_points' unnormalize(points, R, R): k = (R - 1) / R formed in double and rounded once, m = R - 1
  fl.lk.grid = grid; fl.lk.gh = grid_h; fl.lk.gw = grid_w;
  fl.lk.k = static_cast<float>(static_cast<double>(R - 1) / R); fl.lk.m = static_cast<float>(R - 1);
  fl.lk.points_out = points_out;
  fl.flip = flip; fl.query_n = query_n;
  auto st = static_cast<cudaStream_t>(stream);
  float* acc = static_cast<float*>(workspace);
  const int64_t pix = static_cast<int64_t>(p.g.hg) * p.g.wg;
  const unsigned blocks = static_cast<unsigned>((pix + 255) / 256);
  if (!splat) {
    composite_grid_kernel<false, false><<<blocks, 256, 0, st>>>(out, nullptr, images, p, pix);
    GG_CHECK_LAUNCH("composite_grid launch");
    return GG_OK;
  }
  cudaError_t e = cudaMemsetAsync(acc, 0, static_cast<size_t>(frame_bytes), st);
  if (e != cudaSuccess) return cuda_fail(e, "splat_lookup_composite_grid workspace memset");
  const int64_t total = N * P;
  const unsigned sblocks = static_cast<unsigned>((total + 63) / 64);
  if (has_alpha) {
    splat_frames_kernel<true, true><<<sblocks, 64, 0, st>>>(acc, query, colors, alpha, p, total, fl);
    GG_CHECK_LAUNCH("splat_frames lookup launch");
    composite_grid_kernel<true, true><<<blocks, 256, 0, st>>>(out, acc, images, p, pix);
  } else {
    splat_frames_kernel<false, true><<<sblocks, 64, 0, st>>>(acc, query, colors, nullptr, p, total, fl);
    GG_CHECK_LAUNCH("splat_frames lookup launch");
    composite_grid_kernel<true, false><<<blocks, 256, 0, st>>>(out, acc, images, p, pix);
  }
  GG_CHECK_LAUNCH("composite_grid launch");
  return GG_OK;
}

}  // extern "C"
