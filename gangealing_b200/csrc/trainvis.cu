// trainvis.cu -- the training visuals' device work (sm_90a): flow colour-wheel grids, per-cluster sums of congealed
// images and min/max-normalised uint8 grids.  Replaces the host side of the reference's utils/vis_tools/training_vis.py:
//   * flow_to_image (flow_vis.py:22-130) runs in numpy on the host; here one reduction launch (the batch's largest flow
//     radius) and one launch that writes the colour-wheel images straight into make_grid's uint8 layout;
//   * generate_cluster_congeal / real_cluster_congeal (training_vis.py:57-109) move every assigned image to the host with
//     its own .cpu() and sum there; here the images are summed per cluster on the device, in the order they arrive, and
//     only the first n_keep images of each cluster are copied (the grids show n_sample of them);
//   * the per-cluster means' make_grid(normalize=True, range=None, scale_each=True) + images2grid is one launch.
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "grid.cuh"

namespace gg {
namespace {

// ------------------------------------------------------------------------------------------------------ colour wheel
// make_colorwheel (flow_vis.py:22-69): 55 entries, RY 15, YG 6, GC 4, CB 11, BM 13, MR 6; every entry an integer in
// [0, 255] (np.floor(255 * i / n) of exact integers).
constexpr int kNcols = 55;

__device__ __forceinline__ void wheel(int k, double (&c)[3]) {
  int s, n;
  if (k < 15) { s = 0; n = 15; }
  else if (k < 21) { s = 1; n = 6; k -= 15; }
  else if (k < 25) { s = 2; n = 4; k -= 21; }
  else if (k < 36) { s = 3; n = 11; k -= 25; }
  else if (k < 49) { s = 4; n = 13; k -= 36; }
  else { s = 5; n = 6; k -= 49; }
  const double up = floor(255.0 * k / n), down = 255.0 - up;
  switch (s) {
    case 0: c[0] = 255; c[1] = up; c[2] = 0; break;        // RY
    case 1: c[0] = down; c[1] = 255; c[2] = 0; break;      // YG
    case 2: c[0] = 0; c[1] = 255; c[2] = up; break;        // GC
    case 3: c[0] = 0; c[1] = down; c[2] = 255; break;      // CB
    case 4: c[0] = up; c[1] = 0; c[2] = 255; break;        // BM
    default: c[0] = 255; c[1] = 0; c[2] = down; break;     // MR
  }
}

struct FlowParams {
  GridLayout g;
  float scale;            // H - 1: flow_to_image's `flow_uv * (flow_uv.size(1) - 1)`
};

// rad = sqrt(u^2 + v^2) of the scaled flow, in float32 as numpy computes it; the batch maximum by atomicMax on the bit
// pattern (non-negative floats order as their bits do, so the result does not depend on the order).
__global__ void __launch_bounds__(256)
flow_radius_max_kernel(unsigned int* __restrict__ rad_max, const float2* __restrict__ flow, float scale, int64_t total) {
  float m = 0.f;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float2 f = __ldg(flow + i);
    const float u = __fmul_rn(f.x, scale), v = __fmul_rn(f.y, scale);
    m = fmaxf(m, __fsqrt_rn(__fadd_rn(__fmul_rn(u, u), __fmul_rn(v, v))));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(rad_max, __float_as_uint(m));
}

// One grid pixel (3 bytes) per thread: flow_uv_to_colors of the normalised flow with numpy's precision -- float32 up to
// fk (numpy keeps float32 arrays float32, and float32 op Python scalar stays float32), float64 from f = fk - k0 on
// (float32 minus the int32 array k0 promotes to float64, and the wheel is float64), then floor(255 * col).
// The reference divides by 255, lays the images out with make_grid(range=(0, 1)) and quantises with *255 + 0.5: that
// returns floor(255 * col) exactly (the float32 round trip moves it by less than 0.5), so that value is written here.
// arctan2 is evaluated in double and rounded once: the correctly rounded float32 atan2.
__global__ void __launch_bounds__(256)
flow_image_grid_kernel(unsigned char* __restrict__ out, const float2* __restrict__ flow,
                       const unsigned int* __restrict__ rad_max, FlowParams p, int64_t total) {
  const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int gx = static_cast<int>(idx % p.g.wg), gy = static_cast<int>(idx / p.g.wg);
  unsigned char* o = out + idx * 3;
  int y, x;
  const int64_t k = grid_source(p.g, gx, gy, y, x);
  if (k < 0) {
    o[0] = o[1] = o[2] = 0;
    return;
  }
  const float2 f = __ldg(flow + (k * p.g.h + y) * static_cast<int64_t>(p.g.w) + x);
  const float den = __fadd_rn(__uint_as_float(__ldg(rad_max)), 1e-5f);      // rad_max + epsilon
  const float u = __fdiv_rn(__fmul_rn(f.x, p.scale), den), v = __fdiv_rn(__fmul_rn(f.y, p.scale), den);
  const float rad = __fsqrt_rn(__fadd_rn(__fmul_rn(u, u), __fmul_rn(v, v)));
  const float a = __fdiv_rn(static_cast<float>(atan2(-static_cast<double>(v), -static_cast<double>(u))),
                            3.14159265358979323846f);                            // np.arctan2(-v, -u) / np.pi
  const float fk = __fmul_rn(__fdiv_rn(__fadd_rn(a, 1.f), 2.f), static_cast<float>(kNcols - 1));
  const int k0 = static_cast<int>(floorf(fk));
  const int k1 = k0 + 1 == kNcols ? 0 : k0 + 1;
  const double fr = __dsub_rn(static_cast<double>(fk), static_cast<double>(k0));
  double c0[3], c1[3];
  wheel(k0, c0);
  wheel(k1, c1);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    // every double operation rounded on its own, as numpy evaluates it (no contraction into fma)
    double col = __dadd_rn(__dmul_rn(__dsub_rn(1.0, fr), __ddiv_rn(c0[i], 255.0)), __dmul_rn(fr, __ddiv_rn(c1[i], 255.0)));
    col = rad <= 1.f ? __dsub_rn(1.0, __dmul_rn(static_cast<double>(rad), __dsub_rn(1.0, col))) : __dmul_rn(col, 0.75);
    o[i] = static_cast<unsigned char>(static_cast<int>(floor(__dmul_rn(255.0, col))));
  }
}

// ------------------------------------------------------------------------------------------------- per-image ranges
// make_grid(normalize=True, value_range or per-image min/max) + images2grid: one grid pixel (3 bytes) per thread.
__global__ void __launch_bounds__(256)
image_grid_kernel(unsigned char* __restrict__ out, const float* __restrict__ images, const float2* __restrict__ ranges,
                  GridLayout g, int64_t total) {
  const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int gx = static_cast<int>(idx % g.wg), gy = static_cast<int>(idx / g.wg);
  unsigned char* o = out + idx * 3;
  int y, x;
  const int64_t k = grid_source(g, gx, gy, y, x);
  if (k < 0) {
    o[0] = o[1] = o[2] = 0;
    return;
  }
  const int64_t plane = static_cast<int64_t>(g.h) * g.w;
  const float* img = images + k * 3 * plane + static_cast<int64_t>(y) * g.w + x;
  const float2 r = __ldg(ranges + k);
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c] = quantise_range(__ldg(img + c * plane), r.x, r.y);
}

// ------------------------------------------------------------------------------------------------ cluster routing
struct RouteParams {
  int64_t n;                        // images in this call
  int s, k;                         // slots per image (K or 2K), clusters
  int c, h, w;
  int64_t sn, sf, sk, sc, sh, sw;   // element strides: image, flip (slot / K), head (slot % K), channel, row, column
  int n_keep;
};

constexpr int kRouteThreads = 256, kSelChunk = 1024;

// Thread (element e of C*H*W, cluster k): walks the images in order and, for each one routed to k, adds its element to
// the running fp32 sum (one add per image, in order: the sequential sum, bitwise) and copies it into the next keep slot
// while the cluster holds fewer than n_keep.  counts[k] (the images routed to k by earlier calls) is read here and
// advanced by route_count_kernel afterwards, so the fill position carries across calls.
__global__ void __launch_bounds__(kRouteThreads)
route_sum_kernel(float* __restrict__ sums, float* __restrict__ keep, const int64_t* __restrict__ counts,
                 const float* __restrict__ images, const int64_t* __restrict__ sel, RouteParams p) {
  __shared__ int64_t sel_s[kSelChunk];
  const int k = blockIdx.y;
  const int64_t chw = static_cast<int64_t>(p.c) * p.h * p.w;
  const int64_t e = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const bool live = e < chw;
  int c = 0, y = 0, x = 0;
  if (live) {
    x = static_cast<int>(e % p.w);
    y = static_cast<int>((e / p.w) % p.h);
    c = static_cast<int>(e / (static_cast<int64_t>(p.w) * p.h));
  }
  const int64_t off = c * p.sc + y * p.sh + x * p.sw;
  float acc = live ? sums[k * chw + e] : 0.f;
  int64_t filled = counts[k];
  for (int64_t n0 = 0; n0 < p.n; n0 += kSelChunk) {
    const int m = static_cast<int>(p.n - n0 < kSelChunk ? p.n - n0 : kSelChunk);
    __syncthreads();
    for (int i = threadIdx.x; i < m; i += blockDim.x) sel_s[i] = sel[n0 + i];
    __syncthreads();
    for (int i = 0; i < m; ++i) {
      const int64_t s = sel_s[i];
      if (s < 0 || s >= p.s || s % p.k != k) continue;
      if (live) {
        const float v = __ldg(images + (n0 + i) * p.sn + (s / p.k) * p.sf + (s % p.k) * p.sk + off);
        acc = __fadd_rn(acc, v);
        if (filled < p.n_keep) keep[(k * static_cast<int64_t>(p.n_keep) + filled) * chw + e] = v;
      }
      ++filled;
    }
  }
  if (live) sums[k * chw + e] = acc;
}

// counts[k] += the images of this call routed to k (one warp per cluster).
__global__ void route_count_kernel(int64_t* __restrict__ counts, const int64_t* __restrict__ sel, RouteParams p) {
  const int k = blockIdx.x;
  int64_t m = 0;
  for (int64_t i = threadIdx.x; i < p.n; i += 32) {
    const int64_t s = sel[i];
    m += (s >= 0 && s < p.s && s % p.k == k) ? 1 : 0;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m += __shfl_xor_sync(0xffffffffu, m, o);
  if (threadIdx.x == 0) counts[k] += m;
}

inline unsigned blocks_for(int64_t total, int threads) { return static_cast<unsigned>((total + threads - 1) / threads); }

}  // namespace
}  // namespace gg

using namespace gg;

extern "C" {

int gg_flow_image_grid(unsigned char* out, void* workspace, const float* flow, int64_t N, int H, int W, int nrow,
                       int padding, void* stream) {
  GridLayout g;
  if (N < 1 || H < 1 || W < 1 || nrow < 1 || padding < 0)
    return fail(GG_ERR_BAD_ARG, "flow_image_grid: N, H, W, nrow >= 1 and padding >= 0");
  if (!out || !flow || !workspace) return fail(GG_ERR_BAD_ARG, "flow_image_grid: null output, flow or workspace");
  if (!aligned8(flow) || !aligned8(workspace))
    return fail(GG_ERR_BAD_ARG, "flow_image_grid: flow and workspace must be 8-byte aligned (float2 loads)");
  if (!make_grid_layout(g, N, H, W, nrow, padding) || N * H * static_cast<int64_t>(W) > 0x7fffffffLL)
    return fail(GG_ERR_BAD_ARG, "flow_image_grid: the flow or the grid exceeds 2^31 elements");
  auto st = static_cast<cudaStream_t>(stream);
  auto* rad_max = static_cast<unsigned int*>(workspace);
  cudaError_t e = cudaMemsetAsync(rad_max, 0, sizeof(unsigned int), st);
  if (e != cudaSuccess) return cuda_fail(e, "flow_image_grid workspace memset");
  const int64_t pixels = N * H * static_cast<int64_t>(W);
  const int64_t cap = static_cast<int64_t>(sm_count()) * 8;
  const unsigned rb = static_cast<unsigned>(std::min<int64_t>(cap, (pixels + 255) / 256));
  flow_radius_max_kernel<<<rb, 256, 0, st>>>(rad_max, reinterpret_cast<const float2*>(flow), static_cast<float>(H - 1), pixels);
  GG_CHECK_LAUNCH("flow_radius_max launch");
  FlowParams p;
  p.g = g;
  p.scale = static_cast<float>(H - 1);
  const int64_t total = static_cast<int64_t>(g.hg) * g.wg;
  flow_image_grid_kernel<<<blocks_for(total, 256), 256, 0, st>>>(out, reinterpret_cast<const float2*>(flow), rad_max, p, total);
  GG_CHECK_LAUNCH("flow_image_grid launch");
  return GG_OK;
}

int gg_image_grid(unsigned char* out, const float* images, const float* ranges, int64_t N, int H, int W, int nrow,
                  int padding, void* stream) {
  GridLayout g;
  if (N < 1 || H < 1 || W < 1 || nrow < 1 || padding < 0)
    return fail(GG_ERR_BAD_ARG, "image_grid: N, H, W, nrow >= 1 and padding >= 0");
  if (!out || !images || !ranges) return fail(GG_ERR_BAD_ARG, "image_grid: null output, images or ranges");
  if (!aligned8(ranges)) return fail(GG_ERR_BAD_ARG, "image_grid: ranges must be 8-byte aligned (float2 loads)");
  if (!make_grid_layout(g, N, H, W, nrow, padding) || N * 3 * H * static_cast<int64_t>(W) > 0x7fffffffLL)
    return fail(GG_ERR_BAD_ARG, "image_grid: the images or the grid exceed 2^31 elements");
  const int64_t total = static_cast<int64_t>(g.hg) * g.wg;
  image_grid_kernel<<<blocks_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      out, images, reinterpret_cast<const float2*>(ranges), g, total);
  GG_CHECK_LAUNCH("image_grid launch");
  return GG_OK;
}

int gg_cluster_accumulate(float* sums, int64_t* counts, float* keep, const float* images, const int64_t* sel, int64_t N,
                          int S, int K, int C, int H, int W, int64_t stride_n, int64_t stride_flip, int64_t stride_head,
                          int64_t stride_c, int64_t stride_h, int64_t stride_w, int n_keep, void* stream) {
  if (N < 0 || K < 1 || S < K || S % K != 0 || C < 1 || H < 1 || W < 1 || n_keep < 0)
    return fail(GG_ERR_BAD_ARG, "cluster_accumulate: N, n_keep >= 0, K, C, H, W >= 1 and S a positive multiple of K");
  if (K > 65535) return fail(GG_ERR_BAD_ARG, "cluster_accumulate: K <= 65535");
  if (!sums || !counts) return fail(GG_ERR_BAD_ARG, "cluster_accumulate: null sums or counts");
  if (n_keep > 0 && !keep) return fail(GG_ERR_BAD_ARG, "cluster_accumulate: null keep with n_keep > 0");
  if (N > 0 && (!images || !sel)) return fail(GG_ERR_BAD_ARG, "cluster_accumulate: null images or selection");
  if (stride_n < 0 || stride_flip < 0 || stride_head < 0 || stride_c < 0 || stride_h < 0 || stride_w < 0)
    return fail(GG_ERR_BAD_ARG, "cluster_accumulate: strides must be >= 0");
  const int64_t chw = static_cast<int64_t>(C) * H * W;
  if (chw > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "cluster_accumulate: C * H * W exceeds 2^31");
  if (N == 0) return GG_OK;
  RouteParams p;
  p.n = N; p.s = S; p.k = K; p.c = C; p.h = H; p.w = W;
  p.sn = stride_n; p.sf = stride_flip; p.sk = stride_head; p.sc = stride_c; p.sh = stride_h; p.sw = stride_w;
  p.n_keep = n_keep;
  auto st = static_cast<cudaStream_t>(stream);
  route_sum_kernel<<<dim3(blocks_for(chw, kRouteThreads), K), kRouteThreads, 0, st>>>(sums, keep, counts, images, sel, p);
  GG_CHECK_LAUNCH("route_sum launch");
  route_count_kernel<<<K, 32, 0, st>>>(counts, sel, p);
  GG_CHECK_LAUNCH("route_count launch");
  return GG_OK;
}

}  // extern "C"
