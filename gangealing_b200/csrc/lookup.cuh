// lookup.cuh -- `uncongeal_points`' grid lookup as a device function, shared by the fused splat (splat.cu) and the
// PCK-Transfer scorer (pck.cu).
#pragma once
#include "common.cuh"

namespace gg {

// LOOKUP (SURVEY.md 8(f) rank 4, reference spatial_transformer.py:141-157 `uncongeal_points` + helpers.py:178-187): the
// points arrive as QUERY coordinates in the congealed frame; their image positions are looked up in the STN's sampling
// grid -- F.grid_sample(grid as a 2-channel image, query, 'border', align_corners=False) -- and un-normalised to pixels
// (spatial_transformer.py:621-623) as the points are loaded, instead of a grid_sample launch + 4 elementwise launches.
struct LookupParams {
  const float* grid;     // (N, gh, gw, 2)
  int gh, gw;
  float k, m;            // unnormalize: ((g / k) / 2 + 0.5) * m,  k = (res-1)/res, m = out_res - 1
  float* points_out;     // (N, P, 2) or null: the looked-up pixel coordinates
};

__device__ __forceinline__ float2 lookup_point(const LookupParams& lk, int64_t n, float qx, float qy) {
  // ATen grid_sampler_2d, bilinear, padding_mode=border, align_corners=False
  float ix = ((qx + 1.f) * lk.gw - 1.f) / 2.f, iy = ((qy + 1.f) * lk.gh - 1.f) / 2.f;
  ix = fminf(fmaxf(ix, 0.f), static_cast<float>(lk.gw - 1));
  iy = fminf(fmaxf(iy, 0.f), static_cast<float>(lk.gh - 1));
  const float fx = floorf(ix), fy = floorf(iy);
  const int x0 = static_cast<int>(fx), y0 = static_cast<int>(fy);
  const float wx1 = ix - fx, wx0 = (fx + 1.f) - ix, wy1 = iy - fy, wy0 = (fy + 1.f) - iy;
  const float* g = lk.grid + n * lk.gh * static_cast<int64_t>(lk.gw) * 2;
  float ox = 0.f, oy = 0.f;
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      const int yy = y0 + a, xx = x0 + b;
      if (yy >= 0 && yy < lk.gh && xx >= 0 && xx < lk.gw) {
        const float2 v = __ldg(reinterpret_cast<const float2*>(g + (static_cast<int64_t>(yy) * lk.gw + xx) * 2));
        const float w = (a ? wy1 : wy0) * (b ? wx1 : wx0);
        ox = fmaf(v.x, w, ox); oy = fmaf(v.y, w, oy);
      }
    }
  return make_float2(((ox / lk.k) / 2.f + 0.5f) * lk.m, ((oy / lk.k) / 2.f + 0.5f) * lk.m);
}

}  // namespace gg
