// points.cuh -- the nearest-neighbour search of congeal_points (points.cu) for other kernels of the library (pck.cu).
#pragma once
#include "common.cuh"

namespace gg {

// best[n * P + p] = (order-preserving bits of the smallest distance) << 32 | (its grid index, first minimum) for points
// (N, P, 2) against grid (N, HW, 2): the reference's expanded distance |p|^2 + |g|^2 - 2 g.p.  `best` holds N * P
// 64-bit keys.  Launches the search on `st` (two kernels); N * P > 0, HW > 0, N <= 65535 and non-null pointers are the
// caller's to check.
int nn_argmin_search(unsigned long long* best, const float* grid, const float* points, int64_t N, int64_t P, int HW,
                     cudaStream_t st);

}  // namespace gg
