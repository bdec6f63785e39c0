// tv.cuh -- the Huber penalty of total_variation_loss (reference models/losses/loss.py:4-12), shared by the batch-reduced
// training loss (optim.cu) and the per-sample smoothness of flip inference (pck.cu).
#pragma once
#include "common.cuh"

namespace gg {

__device__ __forceinline__ float huber(float d) {            // loss.py:7: where(a <= 1, 0.5 a^2, a - 0.5), a = |d|
  const float a = fabsf(d);
  return a <= 1.f ? 0.5f * a * a : a - 0.5f;
}
__device__ __forceinline__ float huber_grad(float d) {       // d/dd
  return fabsf(d) <= 1.f ? d : (d > 0.f ? 1.f : -1.f);
}

}  // namespace gg
