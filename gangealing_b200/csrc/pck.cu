// pck.cu -- PCK-Transfer evaluation kernels (sm_90a).
//
//   gg_tv_per_sample   reference models/losses/loss.py:4-12 `total_variation_loss(flow, reduce_batch=False)`, the smoothness
//                      that decides every flip of `match_flows` (spatial_transformer.py:270-273) and the score of
//                      applications/flow_scores.py:36.  The tensor formulation is ~10 ATen launches; here ONE launch, one
//                      CTA per sample, a fixed-order block reduction and no atomics: bitwise reproducible.
//   gg_pck_transfer    one transfer direction of applications/pck.py:145-166 for a batch -- ComposedSTN.transfer_points
//                      (spatial_transformer.py:159-198 -> :631-672, :141-157) plus the PCK test -- on the similarity matrix,
//                      residual flow and sampling grid the evaluator already holds from its single STN forward:
//                        1. query   q = normalize(p, S, S) -> inverse similarity (analytic 2x2 inverse, no torch.inverse
//                                   host sync) -> unnormalize(., S, S) -> normalize(., S, S)       (:641-651, :169-178)
//                        2. search  argmin over (delta + identity) of the expanded distance (points.cu, :657-668)
//                        3. score   unravel_index -> normalize(idx, S, F) -> bilinear 'border' lookup in the destination's
//                                   composed grid -> unnormalize(., S, S) (lookup.cuh, :147-153); err = |est - gt|;
//                                   count err <= alpha * thresh (inclusive, pck.py:155) where visible, per alpha
//                      Without a flow (similarity-only SpatialTransformer, :644-651, :692-696) congeal and uncongeal are both
//                      closed-form and step 2 is skipped.  Counts are integer atomics (order-independent: deterministic).
#include "common.cuh"
#include "lookup.cuh"
#include "points.cuh"
#include "tv.cuh"

namespace gg {
namespace {

constexpr int kTvSampleThreads = 512;
constexpr int kPckThreads = 256;
constexpr int kMaxAlphas = 8;

__global__ void __launch_bounds__(kTvSampleThreads)
tv_per_sample_kernel(float* __restrict__ out, const float* __restrict__ flow, int H, int W, float cnt_y, float cnt_x) {
  __shared__ float red_y[kTvSampleThreads / 32], red_x[kTvSampleThreads / 32];
  const int64_t per = static_cast<int64_t>(H) * W * 2;
  const float* f = flow + blockIdx.x * per;
  float sy = 0.f, sx = 0.f;
  for (int64_t i = threadIdx.x; i < per; i += kTvSampleThreads) {
    const int64_t pix = i >> 1;
    const int x = static_cast<int>(pix % W);
    const int y = static_cast<int>(pix / W);
    const float c = f[i];
    if (y + 1 < H) sy += huber(c - f[i + 2 * W]);
    if (x + 1 < W) sx += huber(c - f[i + 2]);
  }
  sy = warp_sum(sy);
  sx = warp_sum(sx);
  if ((threadIdx.x & 31) == 0) { red_y[threadIdx.x >> 5] = sy; red_x[threadIdx.x >> 5] = sx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float ty = 0.f, tx = 0.f;
#pragma unroll
    for (int i = 0; i < kTvSampleThreads / 32; ++i) { ty += red_y[i]; tx += red_x[i]; }
    out[blockIdx.x] = tx / cnt_x + ty / cnt_y;        // loss.py:12 returns dx + dy
  }
}

// The reference's normalize / unnormalize (spatial_transformer.py:617-623) with its operation order, each step rounded.
__device__ __forceinline__ float normalize1(float v, float out_res_m1, float k) {     // v.div(out_res-1).add(-0.5).mul(2).mul(k)
  return __fmul_rn(__fmul_rn(__fadd_rn(__fdiv_rn(v, out_res_m1), -0.5f), 2.f), k);
}
__device__ __forceinline__ float unnormalize1(float v, float k, float out_res_m1) {   // v.div(k).div(2).add(0.5).mul(out_res-1)
  return __fmul_rn(__fadd_rn(__fdiv_rn(__fdiv_rn(v, k), 2.f), 0.5f), out_res_m1);
}

struct PckParams {
  int64_t B, P;
  int A, F;
  float s_m1, f_m1, ks;          // S - 1, F - 1, (S - 1) / S
  bool flow;
};

// threads [0, B*P): the congealed-frame query of every source point; threads [B*P, B*P + B*F*F): the search grid
// delta + identity (flow mode only)
__global__ void __launch_bounds__(kPckThreads)
pck_query_kernel(float* __restrict__ query, float* __restrict__ nn_grid, const float* __restrict__ points,
                 const float* __restrict__ matrix, const float* __restrict__ delta, const float* __restrict__ identity,
                 PckParams p) {
  const int64_t npts = p.B * p.P;
  const int64_t ff = static_cast<int64_t>(p.F) * p.F * 2;
  const int64_t total = npts + (p.flow ? p.B * ff : 0);
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    if (i >= npts) {
      const int64_t j = i - npts;
      nn_grid[j] = __fadd_rn(delta[j], identity[j % ff]);         // flow_or_matrixA + self.identity_flow (:658)
      continue;
    }
    const int64_t b = i / p.P;
    const float x = normalize1(points[i * 2], p.s_m1, p.ks), y = normalize1(points[i * 2 + 1], p.s_m1, p.ks);
    const float* m = matrix + b * 6;                               // [[a, b, c], [d, e, f]]
    // inverse of [M; 0 0 1] (torch.inverse at :648), analytically in double, rounded to fp32 entries
    const double a = m[0], bb = m[1], c = m[2], d = m[3], e = m[4], f = m[5];
    const double r = 1.0 / (a * e - bb * d);
    const float i00 = static_cast<float>(e * r), i01 = static_cast<float>(-bb * r);
    const float i10 = static_cast<float>(-d * r), i11 = static_cast<float>(a * r);
    const float i02 = static_cast<float>((bb * f - e * c) * r), i12 = static_cast<float>((d * c - a * f) * r);
    float cx = __fadd_rn(__fadd_rn(__fmul_rn(x, i00), __fmul_rn(y, i01)), i02);   // (hom @ inv^T)[..., :2]
    float cy = __fadd_rn(__fadd_rn(__fmul_rn(x, i10), __fmul_rn(y, i11)), i12);
    if (p.flow) {   // composed congeal: the similarity STN un-normalises, the flow STN normalises again (:169-178)
      cx = normalize1(unnormalize1(cx, p.ks, p.s_m1), p.s_m1, p.ks);
      cy = normalize1(unnormalize1(cy, p.ks, p.s_m1), p.s_m1, p.ks);
    }
    query[i * 2] = cx;
    query[i * 2 + 1] = cy;
  }
}

__global__ void __launch_bounds__(kPckThreads)
pck_score_kernel(unsigned long long* __restrict__ counts, float* __restrict__ est_out, int64_t* __restrict__ nn_index,
                 const unsigned long long* __restrict__ best, const float* __restrict__ query,
                 const float* __restrict__ gt, const float* __restrict__ visible, const float* __restrict__ thresh,
                 const float* __restrict__ alphas, const float* __restrict__ matrix_dst, LookupParams lk, PckParams p) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * kPckThreads + threadIdx.x;
  const bool live = i < p.B * p.P;
  unsigned hit[kMaxAlphas] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (live) {
    const int64_t b = i / p.P;
    float2 est;
    if (p.flow) {
      const int idx = static_cast<int>(best[i] & 0xffffffffull);
      const int x = idx % p.F, y = idx / p.F;                      // unravel_index(., (F, F)) -> (x, y)
      if (nn_index) nn_index[i] = idx;
      est = lookup_point(lk, b, normalize1(static_cast<float>(x), p.f_m1, p.ks), normalize1(static_cast<float>(y), p.f_m1, p.ks));
    } else {        // closed-form uncongeal: [q, 1] @ [M; 0 0 1]^T, then unnormalize (:692-696, :705-706)
      const float* m = matrix_dst + b * 6;
      const float qx = query[i * 2], qy = query[i * 2 + 1];
      est.x = unnormalize1(__fadd_rn(__fadd_rn(__fmul_rn(qx, m[0]), __fmul_rn(qy, m[1])), m[2]), p.ks, p.s_m1);
      est.y = unnormalize1(__fadd_rn(__fadd_rn(__fmul_rn(qx, m[3]), __fmul_rn(qy, m[4])), m[5]), p.ks, p.s_m1);
    }
    if (est_out) { est_out[i * 2] = est.x; est_out[i * 2 + 1] = est.y; }
    const float dx = __fsub_rn(est.x, gt[i * 2]), dy = __fsub_rn(est.y, gt[i * 2 + 1]);
    const float err = __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));   // (est - gt).norm(dim=-1)
    const bool vis = visible == nullptr || visible[i] != 0.f;
    const float th = thresh[b];
#pragma unroll
    for (int a = 0; a < kMaxAlphas; ++a)
      if (a < p.A) hit[a] = (vis && err <= __fmul_rn(alphas[a], th)) ? 1u : 0u;   // inclusive, as pck.py:155
  }
#pragma unroll
  for (int a = 0; a < kMaxAlphas; ++a) {
    if (a >= p.A) break;
    const unsigned s = __reduce_add_sync(0xffffffffu, hit[a]);
    if ((threadIdx.x & 31) == 0 && s) atomicAdd(counts + a, static_cast<unsigned long long>(s));
  }
}

}  // namespace
}  // namespace gg

using namespace gg;

extern "C" {

int gg_tv_per_sample(float* out, const float* flow, int64_t N, int H, int W, void* stream) {
  if (N < 1 || H < 0 || W < 0) return fail(GG_ERR_BAD_ARG, "tv_per_sample: N must be positive and sizes non-negative");
  if (H < 2 || W < 2) return fail(GG_ERR_BAD_ARG, "tv_per_sample: the flow needs at least 2 x 2 pixels (the reference's mean of an empty difference is nan)");
  if (!out || !flow) return fail(GG_ERR_BAD_ARG, "tv_per_sample: null tensor");
  if (N > 0x7fffffffLL) return fail(GG_ERR_UNSUPPORTED, "tv_per_sample: batch too large");
  const float cnt_y = static_cast<float>(static_cast<int64_t>(H - 1) * W * 2), cnt_x = static_cast<float>(static_cast<int64_t>(H) * (W - 1) * 2);
  tv_per_sample_kernel<<<static_cast<unsigned>(N), kTvSampleThreads, 0, static_cast<cudaStream_t>(stream)>>>(out, flow, H, W, cnt_y, cnt_x);
  GG_CHECK_LAUNCH("tv_per_sample launch");
  return GG_OK;
}

int64_t gg_pck_transfer_workspace(int64_t B, int64_t P, int F) {
  if (B < 1 || P < 1 || F < 0) return 0;
  return B * P * (8 + 8) + B * static_cast<int64_t>(F) * F * 2 * 4;
}

int gg_pck_transfer(int64_t* counts, float* est_points, int64_t* nn_index, void* workspace, const float* points,
                    const float* gt_points, const float* visible, const float* thresh, const float* alphas,
                    const float* matrix_src, const float* matrix_dst, const float* delta_src, const float* identity,
                    const float* grid_dst, int64_t B, int64_t P, int A, int S, int F, int grid_h, int grid_w, void* stream) {
  if (B < 1 || P < 1) return fail(GG_ERR_BAD_ARG, "pck_transfer: B and P must be positive");
  if (A < 1) return fail(GG_ERR_BAD_ARG, "pck_transfer: at least one alpha");
  if (A > kMaxAlphas) return fail(GG_ERR_UNSUPPORTED, "pck_transfer: at most 8 alphas");
  if (S < 2) return fail(GG_ERR_BAD_ARG, "pck_transfer: image size S must be >= 2");
  if (!counts || !workspace || !points || !gt_points || !thresh || !alphas || !matrix_src)
    return fail(GG_ERR_BAD_ARG, "pck_transfer: null tensor");
  const bool flow = delta_src != nullptr;
  if (flow) {
    if (!identity || !grid_dst) return fail(GG_ERR_BAD_ARG, "pck_transfer: null identity flow or destination grid");
    if (F < 2 || F > 46340) return fail(GG_ERR_BAD_ARG, "pck_transfer: flow size F must be in [2, 46340]");
    if (grid_h != F || grid_w != F)
      return fail(GG_ERR_BAD_ARG, "pck_transfer: destination grid resolution %dx%d disagrees with F = %d", grid_h, grid_w, F);
    if (B > 65535) return fail(GG_ERR_UNSUPPORTED, "pck_transfer: batch > 65535");
  } else if (!matrix_dst) {
    return fail(GG_ERR_BAD_ARG, "pck_transfer: null destination matrix (similarity-only STN)");
  }
  auto st = static_cast<cudaStream_t>(stream);
  PckParams p;
  p.B = B; p.P = P; p.A = A; p.F = flow ? F : 0;
  p.s_m1 = static_cast<float>(S - 1);
  p.f_m1 = static_cast<float>(F - 1);
  p.ks = static_cast<float>(static_cast<double>(S - 1) / S);
  p.flow = flow;
  auto* best = static_cast<unsigned long long*>(workspace);
  float* query = reinterpret_cast<float*>(best + B * P);
  float* nn_grid = query + B * P * 2;
  const int64_t total = B * P + (flow ? B * static_cast<int64_t>(F) * F * 2 : 0);
  const int64_t cap = 8LL * sm_count();
  const int64_t qblocks = (total + kPckThreads - 1) / kPckThreads;
  pck_query_kernel<<<static_cast<unsigned>(qblocks < cap ? qblocks : cap), kPckThreads, 0, st>>>(
      query, nn_grid, points, matrix_src, delta_src, identity, p);
  GG_CHECK_LAUNCH("pck_query launch");
  if (flow) {
    const int rc = nn_argmin_search(best, nn_grid, query, B, P, F * F, st);
    if (rc != GG_OK) return rc;
  }
  LookupParams lk;
  lk.grid = grid_dst; lk.gh = grid_h; lk.gw = grid_w; lk.k = p.ks; lk.m = p.s_m1; lk.points_out = nullptr;
  const int64_t sblocks = (B * P + kPckThreads - 1) / kPckThreads;
  if (sblocks > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "pck_transfer: too many points");
  pck_score_kernel<<<static_cast<unsigned>(sblocks), kPckThreads, 0, st>>>(
      reinterpret_cast<unsigned long long*>(counts), est_points, nn_index, best, query, gt_points, visible, thresh, alphas,
      matrix_dst, lk, p);
  GG_CHECK_LAUNCH("pck_score launch");
  return GG_OK;
}

}  // extern "C"
