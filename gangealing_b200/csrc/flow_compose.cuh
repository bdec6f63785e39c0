// flow_compose.cuh -- the flow head's per-pixel grid composition (reference warping_heads.py:180-193 upsample_flow,
// :239-244, :268-277 apply_affine), shared by the stand-alone op (flow.cu: its forward and the three backward kernels,
// which recompute it) and the one-pass sampler (warp.cu, mode 2), so that every path evaluates the same operations.
#pragma once
#include "common.cuh"

namespace gg {

// RAFT convex up-sampling at full-resolution pixel (h*s + sy, w*s + sx) of sample n: the softmax weights pk of its 9 mask
// logits (mask (N, 9*s*s, lh, lw) viewed (N, 9, s, s, lh, lw)), the 3x3 neighbourhood (fx, fy) of s*low (N, lh, lw, 2)
// (zero padded, F.unfold padding=1) and, returned, their convex combination delta = sum_k pk * (fx, fy).
__device__ __forceinline__ float2 convex_upsample(const float* low, const float* mask, int64_t n, int lh, int lw, int s,
                                                  int sy, int sx, int h, int w, float (&pk)[9], float (&fx)[9],
                                                  float (&fy)[9]) {
  float mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    pk[k] = __ldg(mask + ((((n * 9 + k) * s + sy) * s + sx) * lh + h) * static_cast<int64_t>(lw) + w);
    mx = fmaxf(mx, pk[k]);
  }
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < 9; ++k) { pk[k] = expf(pk[k] - mx); sum += pk[k]; }
  const float inv = 1.f / sum;
  float dx = 0.f, dy = 0.f;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const int hh = h + k / 3 - 1, ww = w + k % 3 - 1;
    pk[k] *= inv;
    fx[k] = 0.f; fy[k] = 0.f;
    if (hh >= 0 && hh < lh && ww >= 0 && ww < lw) {
      const float2 f = __ldg(reinterpret_cast<const float2*>(low + ((n * lh + hh) * static_cast<int64_t>(lw) + ww) * 2));
      fx[k] = static_cast<float>(s) * f.x; fy[k] = static_cast<float>(s) * f.y;
    }
    dx = fmaf(pk[k], fx[k], dx);
    dy = fmaf(pk[k], fy[k], dy);
  }
  return make_float2(dx, dy);
}

// the sampling grid at that pixel: identity + delta, then [gx, gy, 1] @ M^T with the base warp M = base[n] (N, 2, 3)
// and identity.lerp(grid, alpha[n]) = identity + alpha*(grid - identity); base / alpha null: skipped
__device__ __forceinline__ float2 compose_flow(float2 id, float dx, float dy, const float* base, const float* alpha,
                                               int64_t n) {
  float gx = id.x + dx, gy = id.y + dy;
  if (base) {
    const float* M = base + n * 6;
    const float tx = M[0] * gx + M[1] * gy + M[2];
    const float ty = M[3] * gx + M[4] * gy + M[5];
    gx = tx; gy = ty;
  }
  if (alpha) {
    const float a = __ldg(alpha + n);
    gx = id.x + a * (gx - id.x);
    gy = id.y + a * (gy - id.y);
  }
  return make_float2(gx, gy);
}

// blocks of a grid-stride launch: enough for `total` items, at most 16 CTAs per SM
inline int grid_for(int64_t total, int threads) {
  const int64_t g = (total + threads - 1) / threads;
  const int64_t cap = static_cast<int64_t>(sm_count()) * 16;
  return static_cast<int>(g < cap ? (g > 0 ? g : 1) : cap);
}

}  // namespace gg
